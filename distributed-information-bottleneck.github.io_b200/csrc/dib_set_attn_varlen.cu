// dib_set_attn_varlen.cu -- the set-attention core for sets of different sizes (dib_config.variable_set_sizes): every set is
// stored padded to Lmax = set_size rows and set s has l_s = set_sizes[s] real particles.  Keys j >= l_s are masked out of
// every query's softmax (Keras 2 MultiHeadAttention with attention_mask: the masked scores get a large negative addend, so
// with at least one real key their weight is exactly 0 in fp32 -- here they are skipped), and padding query rows produce zero
// outputs and zero gradients.
//
// Key-tiled, so shared memory does not depend on Lmax: one CTA per (head, set, 64-row tile), 64-key tiles with an online
// softmax in the forward; the backward is a dQ pass over the query tiles (which also writes D = rowsum(dO o O) once per row)
// followed by a dK / dV pass over the key tiles.  Tiles at or past l_s are skipped, so the work follows sum_s l_s^2.  Each of
// the 256 threads owns a 4 x 4 micro-tile of the 64 x 64 score tile and a 4 x 8 micro-tile of the 64 x dk output tile in
// registers.  fp32 CUDA-core arithmetic in every precision mode, no atomics, fixed summation order: bit-identical run to run.
#include "dib_common.cuh"
#include "dib_kernels.h"

namespace {

constexpr int kT = 64;            // rows of a query tile and of a key tile
constexpr int kThreads = 256;     // 16 x 16 threads: ty owns tile rows 4 ty .. 4 ty + 3, tx columns tx + 16 j
constexpr int kMaxDk = 128;
constexpr int kOC = kMaxDk / 16;  // output columns per thread
constexpr int kSP = kT + 1;       // pitch of the 64 x 64 score tiles

__device__ __forceinline__ int set_len(const DibAttnArgs& a, long long set) {
  const int l = a.set_sizes[set];
  return l < 1 ? 1 : (l > a.L ? a.L : l);
}

// rows [r0, r0 + kT) of one head of a set into a [kT, dk + 1] tile; rows >= lim are zero
__device__ __forceinline__ void load_tile(float* dst, const float* src, int ld, long long row0, int col0, int r0, int lim, int dk,
                                          float scale) {
  for (int idx = threadIdx.x; idx < kT * dk; idx += kThreads) {
    const int i = idx / dk, d = idx % dk;
    dst[i * (dk + 1) + d] = r0 + i < lim ? src[(row0 + r0 + i) * (long long)ld + col0 + d] * scale : 0.f;
  }
}

// zero rows [r0, min(r0 + kT, L)) of up to two [sets * L, ld] outputs (padding rows of a set)
__device__ __forceinline__ void zero_rows(float* a, float* b, int ld, long long row0, int col0, int r0, int L, int dk) {
  const int rows = L - r0 < kT ? L - r0 : kT;
  for (int idx = threadIdx.x; idx < rows * dk; idx += kThreads) {
    const long long g = (row0 + r0 + idx / dk) * (long long)ld + col0 + idx % dk;
    a[g] = 0.f;
    if (b) b[g] = 0.f;
  }
}

// the 16 threads of a tile row are one half-warp
__device__ __forceinline__ float half_max(float v) {
#pragma unroll
  for (int o = 8; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}
__device__ __forceinline__ float half_sum(float v) {
#pragma unroll
  for (int o = 8; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// acc[i][j] = sum_d A[4 ty + i][d] B[tx + 16 j][d] over two [kT, dk + 1] tiles
__device__ __forceinline__ void tile_dots(float acc[4][4], const float* A, const float* B, int dk, int ty, int tx) {
  const int P1 = dk + 1;
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) acc[i][j] = 0.f;
  for (int d = 0; d < dk; ++d) {
    float av[4], bv[4];
#pragma unroll
    for (int i = 0; i < 4; ++i) av[i] = A[(4 * ty + i) * P1 + d];
#pragma unroll
    for (int j = 0; j < 4; ++j) bv[j] = B[(tx + 16 * j) * P1 + d];
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
      for (int j = 0; j < 4; ++j) acc[i][j] = fmaf(av[i], bv[j], acc[i][j]);
  }
}

// acc[i][c] += sum_{t < tn} W[4 ty + i][t] X[t][tx + 16 c] (W a [kT, kSP] score tile, X a [kT, dk + 1] row tile)
__device__ __forceinline__ void tile_accum(float acc[4][kOC], const float* W, const float* X, int tn, int dk, int tx) {
  const int P1 = dk + 1, ty = threadIdx.x / 16;
  for (int t = 0; t < tn; ++t) {
    float w[4], x[kOC];
#pragma unroll
    for (int i = 0; i < 4; ++i) w[i] = W[(4 * ty + i) * kSP + t];
#pragma unroll
    for (int c = 0; c < kOC; ++c) x[c] = tx + 16 * c < dk ? X[t * P1 + tx + 16 * c] : 0.f;
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
      for (int c = 0; c < kOC; ++c) acc[i][c] = fmaf(w[i], x[c], acc[i][c]);
  }
}

// forward: O = softmax(Q K^T / sqrt(dk) over the l real keys) V and the row log-sum-exp, for one query tile
__global__ void __launch_bounds__(kThreads)
attn_varlen_fwd_kernel(DibAttnArgs a) {
  extern __shared__ float sm[];
  const int dk = a.dk, hd = blockIdx.x, P1 = dk + 1, q0 = blockIdx.z * kT;
  const long long set = blockIdx.y, row0 = set * a.L;
  const int col0 = hd * dk, l = set_len(a, set);
  float* lse = a.lse + (set * gridDim.x + hd) * a.L;
  if (q0 >= l) {                                  // a tile of padding rows
    zero_rows(a.o, nullptr, a.ld, row0, col0, q0, a.L, dk);
    for (int i = threadIdx.x; i < kT && q0 + i < a.L; i += kThreads) lse[q0 + i] = 0.f;
    return;
  }
  float* Qs = sm;
  float* Ks = Qs + kT * P1;
  float* Vs = Ks + kT * P1;
  float* Ps = Vs + kT * P1;
  const int tx = threadIdx.x % 16, ty = threadIdx.x / 16;
  load_tile(Qs, a.q, a.ld, row0, col0, q0, l, dk, 1.f / sqrtf((float)dk));
  float m[4], lsum[4], o[4][kOC];
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    m[i] = -INFINITY; lsum[i] = 0.f;
#pragma unroll
    for (int c = 0; c < kOC; ++c) o[i][c] = 0.f;
  }
  for (int k0 = 0; k0 < l; k0 += kT) {
    __syncthreads();                              // the previous tile's K / V / P are consumed
    load_tile(Ks, a.k, a.ld, row0, col0, k0, l, dk, 1.f);
    load_tile(Vs, a.v, a.ld, row0, col0, k0, l, dk, 1.f);
    __syncthreads();
    float s[4][4];
    tile_dots(s, Qs, Ks, dk, ty, tx);
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      float mt = -INFINITY;
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        if (k0 + tx + 16 * j >= l) s[i][j] = -INFINITY;     // masked key
        mt = fmaxf(mt, s[i][j]);
      }
      const float mn = fmaxf(m[i], half_max(mt));           // finite: key k0 is real
      const float alpha = expf(m[i] - mn);
      float ps = 0.f;
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const float p = expf(s[i][j] - mn);
        Ps[(4 * ty + i) * kSP + tx + 16 * j] = p;
        ps += p;
      }
      lsum[i] = fmaf(lsum[i], alpha, half_sum(ps));
      m[i] = mn;
#pragma unroll
      for (int c = 0; c < kOC; ++c) o[i][c] *= alpha;
    }
    __syncthreads();
    tile_accum(o, Ps, Vs, l - k0 < kT ? l - k0 : kT, dk, tx);
  }
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int r = q0 + 4 * ty + i;
    if (r >= a.L) continue;
    const bool real = r < l;
    const float inv = 1.f / lsum[i];
#pragma unroll
    for (int c = 0; c < kOC; ++c) {
      const int d = tx + 16 * c;
      if (d < dk) a.o[(row0 + r) * (long long)a.ld + col0 + d] = real ? dib_maybe_round(o[i][c] * inv, a.round_out) : 0.f;
    }
    if (tx == 0) lse[r] = real ? m[i] + logf(lsum[i]) : 0.f;
  }
}

// backward, query side: D = rowsum(dO o O) of the tile's rows (kept for the key pass), then over the key tiles
//   P = exp(S - lse), dP = dO V^T, dS = P o (dP - D), dQ += dS K;  dQ / sqrt(dk) out
__global__ void __launch_bounds__(kThreads)
attn_varlen_bwd_dq_kernel(DibAttnArgs a) {
  extern __shared__ float sm[];
  const int dk = a.dk, hd = blockIdx.x, P1 = dk + 1, q0 = blockIdx.z * kT;
  const long long set = blockIdx.y, row0 = set * a.L;
  const int col0 = hd * dk, l = set_len(a, set);
  const long long hrow = (set * gridDim.x + hd) * a.L;
  if (q0 >= l) {
    zero_rows(a.dq, nullptr, a.ld, row0, col0, q0, a.L, dk);
    for (int i = threadIdx.x; i < kT && q0 + i < a.L; i += kThreads) a.dsum[hrow + q0 + i] = 0.f;
    return;
  }
  float* Qs = sm;
  float* dOs = Qs + kT * P1;
  float* Ks = dOs + kT * P1;
  float* Vs = Ks + kT * P1;
  float* dSs = Vs + kT * P1;
  float* Dr = dSs + kT * kSP;
  float* Lr = Dr + kT;
  const int tx = threadIdx.x % 16, ty = threadIdx.x / 16, warp = threadIdx.x / 32, lane = threadIdx.x % 32;
  const float scale = 1.f / sqrtf((float)dk);
  load_tile(Qs, a.q, a.ld, row0, col0, q0, l, dk, scale);
  load_tile(dOs, a.dout, a.ld, row0, col0, q0, l, dk, 1.f);
  __syncthreads();
  for (int i = warp; i < kT; i += kThreads / 32) {
    const int r = q0 + i;
    float t = 0.f;
    if (r < l) {
      const float* o = a.o + (row0 + r) * (long long)a.ld + col0;
      for (int d = lane; d < dk; d += 32) t = fmaf(dOs[i * P1 + d], o[d], t);
    }
    t = dib_warp_sum(t);
    if (lane == 0) {
      Dr[i] = t;
      Lr[i] = r < l ? a.lse[hrow + r] : 0.f;
      if (r < a.L) a.dsum[hrow + r] = t;
    }
  }
  float dq[4][kOC];
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int c = 0; c < kOC; ++c) dq[i][c] = 0.f;
  for (int k0 = 0; k0 < l; k0 += kT) {
    __syncthreads();
    load_tile(Ks, a.k, a.ld, row0, col0, k0, l, dk, 1.f);
    load_tile(Vs, a.v, a.ld, row0, col0, k0, l, dk, 1.f);
    __syncthreads();
    float s[4][4], dp[4][4];
    tile_dots(s, Qs, Ks, dk, ty, tx);
    tile_dots(dp, dOs, Vs, dk, ty, tx);
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const int r = 4 * ty + i;
      const bool rr = q0 + r < l;
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const float p = rr && k0 + tx + 16 * j < l ? expf(s[i][j] - Lr[r]) : 0.f;
        dSs[r * kSP + tx + 16 * j] = p * (dp[i][j] - Dr[r]);
      }
    }
    __syncthreads();
    tile_accum(dq, dSs, Ks, l - k0 < kT ? l - k0 : kT, dk, tx);
  }
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int r = q0 + 4 * ty + i;
    if (r >= a.L) continue;
#pragma unroll
    for (int c = 0; c < kOC; ++c) {
      const int d = tx + 16 * c;
      if (d < dk) a.dq[(row0 + r) * (long long)a.ld + col0 + d] = r < l ? dib_maybe_round(dq[i][c] * scale, a.round_out) : 0.f;
    }
  }
}

// backward, key side: over the query tiles, with the key tile's K / V resident,
//   P^T, dS^T as in the query pass;  dV += P^T dO,  dK += dS^T Q / sqrt(dk)
__global__ void __launch_bounds__(kThreads)
attn_varlen_bwd_dkdv_kernel(DibAttnArgs a) {
  extern __shared__ float sm[];
  const int dk = a.dk, hd = blockIdx.x, P1 = dk + 1, k0 = blockIdx.z * kT;
  const long long set = blockIdx.y, row0 = set * a.L;
  const int col0 = hd * dk, l = set_len(a, set);
  const long long hrow = (set * gridDim.x + hd) * a.L;
  if (k0 >= l) {
    zero_rows(a.dk_, a.dv, a.ld, row0, col0, k0, a.L, dk);
    return;
  }
  float* Ks = sm;
  float* Vs = Ks + kT * P1;
  float* Qs = Vs + kT * P1;
  float* dOs = Qs + kT * P1;
  float* Pt = dOs + kT * P1;
  float* dSt = Pt + kT * kSP;
  float* Dr = dSt + kT * kSP;
  float* Lr = Dr + kT;
  const int tx = threadIdx.x % 16, ty = threadIdx.x / 16;
  const float scale = 1.f / sqrtf((float)dk);
  load_tile(Ks, a.k, a.ld, row0, col0, k0, l, dk, 1.f);
  load_tile(Vs, a.v, a.ld, row0, col0, k0, l, dk, 1.f);
  float dkk[4][kOC], dv[4][kOC];
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int c = 0; c < kOC; ++c) dkk[i][c] = dv[i][c] = 0.f;
  for (int q0 = 0; q0 < l; q0 += kT) {
    __syncthreads();
    load_tile(Qs, a.q, a.ld, row0, col0, q0, l, dk, scale);
    load_tile(dOs, a.dout, a.ld, row0, col0, q0, l, dk, 1.f);
    for (int i = threadIdx.x; i < kT; i += kThreads) {
      const bool rr = q0 + i < l;
      Dr[i] = rr ? a.dsum[hrow + q0 + i] : 0.f;
      Lr[i] = rr ? a.lse[hrow + q0 + i] : 0.f;
    }
    __syncthreads();
    float s[4][4], dp[4][4];              // [key 4 ty + i][query tx + 16 j]
    tile_dots(s, Ks, Qs, dk, ty, tx);
    tile_dots(dp, Vs, dOs, dk, ty, tx);
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const int kr = 4 * ty + i;
      const bool kreal = k0 + kr < l;
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const int qc = tx + 16 * j;
        const float p = kreal && q0 + qc < l ? expf(s[i][j] - Lr[qc]) : 0.f;
        Pt[kr * kSP + qc] = p;
        dSt[kr * kSP + qc] = p * (dp[i][j] - Dr[qc]);
      }
    }
    __syncthreads();
    const int tn = l - q0 < kT ? l - q0 : kT;
    tile_accum(dv, Pt, dOs, tn, dk, tx);
    tile_accum(dkk, dSt, Qs, tn, dk, tx);
  }
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int r = k0 + 4 * ty + i;
    if (r >= a.L) continue;
    const bool real = r < l;
#pragma unroll
    for (int c = 0; c < kOC; ++c) {
      const int d = tx + 16 * c;
      if (d >= dk) continue;
      const long long g = (row0 + r) * (long long)a.ld + col0 + d;
      a.dk_[g] = real ? dib_maybe_round(dkk[i][c], a.round_out) : 0.f;
      a.dv[g] = real ? dib_maybe_round(dv[i][c], a.round_out) : 0.f;
    }
  }
}

// pooled[s, e] = (sum_{p < l_s} x[s Lmax + p, e]) / l_s
__global__ void pool_varlen_fwd_kernel(const float* x, int ld, int E, int Lmax, long long sets, const int* sizes, float* out,
                                       int ldo, int round_out) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= sets * ldo) return;
  const long long s = i / ldo;
  const int e = (int)(i % ldo);
  int l = sizes[s];
  l = l < 1 ? 1 : (l > Lmax ? Lmax : l);
  float acc = 0.f;
  if (e < E)
    for (int p = 0; p < l; ++p) acc += x[(s * Lmax + p) * ld + e];
  out[i] = e < E ? dib_maybe_round(acc / (float)l, round_out) : 0.f;
}

// every column of the padding rows p >= l_s of a [sets * Lmax, ld] buffer set to zero
__global__ void zero_pad_rows_kernel(float* buf, int ld, long long rows, int Lmax, const int* sizes) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= rows * ld) return;
  const long long r = i / ld, s = r / Lmax;
  if ((int)(r - s * Lmax) >= sizes[s]) buf[i] = 0.f;
}

size_t smem_fwd(int dk) { return sizeof(float) * (3 * kT * (dk + 1) + kT * kSP); }
size_t smem_dq(int dk) { return sizeof(float) * (4 * kT * (dk + 1) + kT * kSP + 2 * kT); }
size_t smem_dkdv(int dk) { return sizeof(float) * (4 * kT * (dk + 1) + 2 * kT * kSP + 2 * kT); }

dim3 grid_of(const DibAttnArgs& a) { return dim3(a.heads, (unsigned)a.sets, (unsigned)DIB_CEIL_DIV(a.L, kT)); }

}  // namespace

// shared memory depends on dk only (<= 157 KB at dk = 128); the opt-in at dk = 128, once per model creation
cudaError_t dib_attn_varlen_prepare() {
  cudaError_t e = cudaFuncSetAttribute(attn_varlen_fwd_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_fwd(kMaxDk));
  if (e == cudaSuccess)
    e = cudaFuncSetAttribute(attn_varlen_bwd_dq_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_dq(kMaxDk));
  if (e == cudaSuccess)
    e = cudaFuncSetAttribute(attn_varlen_bwd_dkdv_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_dkdv(kMaxDk));
  return e;
}

cudaError_t dib_launch_attn_varlen_fwd(const DibAttnArgs& a, cudaStream_t st) {
  if (a.sets == 0) return cudaSuccess;
  attn_varlen_fwd_kernel<<<grid_of(a), kThreads, smem_fwd(a.dk), st>>>(a);
  dib_note_launch();
  return cudaGetLastError();
}

cudaError_t dib_launch_attn_varlen_bwd(const DibAttnArgs& a, cudaStream_t st) {
  if (a.sets == 0) return cudaSuccess;
  attn_varlen_bwd_dq_kernel<<<grid_of(a), kThreads, smem_dq(a.dk), st>>>(a);
  dib_note_launch();
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return e;
  attn_varlen_bwd_dkdv_kernel<<<grid_of(a), kThreads, smem_dkdv(a.dk), st>>>(a);
  dib_note_launch();
  return cudaGetLastError();
}

cudaError_t dib_launch_pool_varlen_fwd(const float* x, int ld, int E, int Lmax, int64_t sets, const int* sizes, float* out, int ldo,
                                       int round_out, cudaStream_t st) {
  const long long count = sets * ldo;
  if (count == 0) return cudaSuccess;
  pool_varlen_fwd_kernel<<<(unsigned)DIB_CEIL_DIV(count, 256ll), 256, 0, st>>>(x, ld, E, Lmax, sets, sizes, out, ldo, round_out);
  dib_note_launch();
  return cudaGetLastError();
}

cudaError_t dib_launch_zero_pad_rows(float* buf, int ld, int64_t rows, int Lmax, const int* sizes, cudaStream_t st) {
  const long long count = rows * ld;
  if (count == 0) return cudaSuccess;
  zero_pad_rows_kernel<<<(unsigned)DIB_CEIL_DIV(count, 256ll), 256, 0, st>>>(buf, ld, rows, Lmax, sizes);
  dib_note_launch();
  return cudaGetLastError();
}
