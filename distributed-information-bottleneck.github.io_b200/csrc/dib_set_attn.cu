// dib_set_attn.cu -- the set-attention integration network of nb-particle cell 8 (dib_config.integration_kind = 1): the
// attention core of Keras 2's MultiHeadAttention (no dropout, no mask), residual + LayerNormalization, and the mean over
// the particles of a set, forward and backward.  The dense projections around them (Q / K / V, output, feed-forward,
// head) run on the grouped GEMMs of dib_gemm_simt.cu / dib_gemm_tc.cu; everything here is fp32 CUDA-core arithmetic in
// every precision mode.  Every reduction has a fixed order and no kernel uses atomics, so results are bit-identical run
// to run.
#include "dib_common.cuh"
#include "dib_kernels.h"

namespace {

constexpr int kAttnThreads = 256;

// Q / K / V (and dO) of one (set, head) in shared memory: L rows of dk floats with a row pitch of dk + 1, so that the
// lanes of a warp reading column d of consecutive rows hit distinct banks
__device__ __forceinline__ void load_rows(float* dst, const float* src, int ld, long long row0, int col0, int L, int dk,
                                          float scale, int nthreads) {
  for (int idx = threadIdx.x; idx < L * dk; idx += nthreads) {
    const int i = idx / dk, d = idx % dk;
    dst[i * (dk + 1) + d] = src[(row0 + i) * (long long)ld + col0 + d] * scale;
  }
}

// S = (Q/sqrt(dk)) K^T [L x L], pitch L + 1
__device__ __forceinline__ void scores(float* S, const float* Qs, const float* Ks, int L, int dk) {
  for (int idx = threadIdx.x; idx < L * L; idx += kAttnThreads) {
    const int i = idx / L, j = idx % L;
    const float* q = Qs + i * (dk + 1);
    const float* k = Ks + j * (dk + 1);
    float s = 0.f;
    for (int d = 0; d < dk; ++d) s = fmaf(q[d], k[d], s);
    S[i * (L + 1) + j] = s;
  }
}

// one CTA per (head, set): S, the max-subtracted row softmax P (kept in shared memory only), O = P V, and the row
// log-sum-exp m_i + log(sum_j exp(S_ij - m_i)) that the backward recomputes P from
__global__ void __launch_bounds__(kAttnThreads)
attn_fwd_kernel(DibAttnArgs a) {
  extern __shared__ float sm[];
  const int L = a.L, dk = a.dk, hd = blockIdx.x, set = blockIdx.y, P1 = dk + 1;
  float* Qs = sm;
  float* Ks = Qs + L * P1;
  float* Vs = Ks + L * P1;
  float* S = Vs + L * P1;
  const long long row0 = (long long)set * L;
  const int col0 = hd * dk;
  const float scale = 1.f / sqrtf((float)dk);
  load_rows(Qs, a.q, a.ld, row0, col0, L, dk, scale, kAttnThreads);
  load_rows(Ks, a.k, a.ld, row0, col0, L, dk, 1.f, kAttnThreads);
  load_rows(Vs, a.v, a.ld, row0, col0, L, dk, 1.f, kAttnThreads);
  __syncthreads();
  scores(S, Qs, Ks, L, dk);
  __syncthreads();
  const int warp = threadIdx.x / 32, lane = threadIdx.x % 32;
  for (int i = warp; i < L; i += kAttnThreads / 32) {
    float* s = S + i * (L + 1);
    float m = -INFINITY;
    for (int j = lane; j < L; j += 32) m = fmaxf(m, s[j]);
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
    float sum = 0.f;
    for (int j = lane; j < L; j += 32) { const float e = expf(s[j] - m); s[j] = e; sum += e; }
    sum = dib_warp_sum(sum);
    const float inv = 1.f / sum;
    for (int j = lane; j < L; j += 32) s[j] *= inv;
    if (lane == 0) a.lse[((long long)set * gridDim.x + hd) * L + i] = m + logf(sum);
  }
  __syncthreads();
  for (int idx = threadIdx.x; idx < L * dk; idx += kAttnThreads) {
    const int i = idx / dk, d = idx % dk;
    const float* p = S + i * (L + 1);
    float o = 0.f;
    for (int j = 0; j < L; ++j) o = fmaf(p[j], Vs[j * P1 + d], o);
    a.o[(row0 + i) * (long long)a.ld + col0 + d] = dib_maybe_round(o, a.round_out);
  }
}

// one CTA per (head, set): P from the saved log-sum-exp, then
//   dV = P^T dO,  dP = dO V^T,  dS = P o (dP - rowsum(dO o O)),  dQ = dS K / sqrt(dk),  dK = dS^T Q / sqrt(dk)
__global__ void __launch_bounds__(kAttnThreads)
attn_bwd_kernel(DibAttnArgs a) {
  extern __shared__ float sm[];
  const int L = a.L, dk = a.dk, hd = blockIdx.x, set = blockIdx.y, P1 = dk + 1;
  float* Qs = sm;
  float* Ks = Qs + L * P1;
  float* Vs = Ks + L * P1;
  float* dOs = Vs + L * P1;
  float* S = dOs + L * P1;        // P
  float* dS = S + L * (L + 1);
  float* Dr = dS + L * (L + 1);   // rowsum(dO o O)
  const long long row0 = (long long)set * L;
  const int col0 = hd * dk;
  const float scale = 1.f / sqrtf((float)dk);
  load_rows(Qs, a.q, a.ld, row0, col0, L, dk, scale, kAttnThreads);
  load_rows(Ks, a.k, a.ld, row0, col0, L, dk, 1.f, kAttnThreads);
  load_rows(Vs, a.v, a.ld, row0, col0, L, dk, 1.f, kAttnThreads);
  load_rows(dOs, a.dout, a.ld, row0, col0, L, dk, 1.f, kAttnThreads);
  __syncthreads();
  scores(S, Qs, Ks, L, dk);
  const int warp = threadIdx.x / 32, lane = threadIdx.x % 32;
  for (int i = warp; i < L; i += kAttnThreads / 32) {
    const float* o = a.o + (row0 + i) * (long long)a.ld + col0;
    float t = 0.f;
    for (int d = lane; d < dk; d += 32) t = fmaf(dOs[i * P1 + d], o[d], t);
    t = dib_warp_sum(t);
    if (lane == 0) Dr[i] = t;
  }
  __syncthreads();
  const float* lse = a.lse + ((long long)set * gridDim.x + hd) * L;
  for (int idx = threadIdx.x; idx < L * L; idx += kAttnThreads) {
    const int i = idx / L, j = idx % L;
    const float p = expf(S[i * (L + 1) + j] - lse[i]);
    const float* g = dOs + i * P1;
    const float* v = Vs + j * P1;
    float dp = 0.f;
    for (int d = 0; d < dk; ++d) dp = fmaf(g[d], v[d], dp);
    S[i * (L + 1) + j] = p;
    dS[i * (L + 1) + j] = p * (dp - Dr[i]);
  }
  __syncthreads();
  for (int idx = threadIdx.x; idx < L * dk; idx += kAttnThreads) {
    const int r = idx / dk, d = idx % dk;
    float dv = 0.f, dq = 0.f, dkk = 0.f;
    for (int t = 0; t < L; ++t) {
      dv = fmaf(S[t * (L + 1) + r], dOs[t * P1 + d], dv);
      dq = fmaf(dS[r * (L + 1) + t], Ks[t * P1 + d], dq);
      dkk = fmaf(dS[t * (L + 1) + r], Qs[t * P1 + d], dkk);
    }
    const long long g = (row0 + r) * (long long)a.ld + col0 + d;
    a.dv[g] = dib_maybe_round(dv, a.round_out);
    a.dq[g] = dib_maybe_round(dq * scale, a.round_out);
    a.dk_[g] = dib_maybe_round(dkk, a.round_out);
  }
}

constexpr int kLnWarps = 8;

// z = a + b, y = (z - mean) * rstd * gamma + beta with the biased variance (Keras LayerNormalization, axis -1); one warp
// per row, columns lane, lane + 32, ... (E <= 128)
__global__ void __launch_bounds__(kLnWarps * 32)
ln_fwd_kernel(DibLayerNorm a) {
  const int lane = threadIdx.x % 32, E = a.E;
  const long long r = (long long)blockIdx.x * kLnWarps + threadIdx.x / 32;
  if (r >= a.rows) return;
  float z[4];
  float s = 0.f;
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    const int e = lane + 32 * k;
    z[k] = e < E ? a.a[r * a.ld + e] + a.b[r * a.ld + e] : 0.f;
    s += z[k];
  }
  const float mean = dib_warp_sum(s) / (float)E;
  float v = 0.f;
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    const int e = lane + 32 * k;
    const float c = e < E ? z[k] - mean : 0.f;
    v = fmaf(c, c, v);
  }
  const float rstd = 1.f / sqrtf(dib_warp_sum(v) / (float)E + a.epsilon);
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    const int e = lane + 32 * k;
    if (e < E) a.y[r * a.ld + e] = dib_maybe_round((z[k] - mean) * rstd * a.gamma[e] + a.beta[e], a.round_out);
    else if (e < a.ld) a.y[r * a.ld + e] = 0.f;
  }
  if (lane == 0) { a.mean[r] = mean; a.rstd[r] = rstd; }
}

// dy = sum of the per-row sources (+ the pooled source / L); dz = rstd (dy g - mean(dy g) - xhat mean(dy g xhat)).
// CTA s owns rows [s * rows_per_split, ...) and writes its d gamma / d beta partials to row s of the split table.
__global__ void __launch_bounds__(kLnWarps * 32)
ln_bwd_kernel(DibLayerNorm a, DibLayerNormBwd b) {
  __shared__ float red[kLnWarps][2][128];
  const int lane = threadIdx.x % 32, warp = threadIdx.x / 32, E = a.E;
  const long long r0 = (long long)blockIdx.x * b.rows_per_split;
  const long long r1 = r0 + b.rows_per_split < a.rows ? r0 + b.rows_per_split : a.rows;
  float dg[4] = {0.f, 0.f, 0.f, 0.f}, db[4] = {0.f, 0.f, 0.f, 0.f};
  for (long long r = r0 + warp; r < r1; r += kLnWarps) {
    const float mean = a.mean[r], rstd = a.rstd[r];
    float xh[4], g[4];
    float s1 = 0.f, s2 = 0.f;
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const int e = lane + 32 * k;
      xh[k] = g[k] = 0.f;
      if (e >= E) continue;
      xh[k] = (a.a[r * a.ld + e] + a.b[r * a.ld + e] - mean) * rstd;
      float dy = 0.f;
      if (b.dy_pool && b.set_sizes) {          // padded sets of different sizes: the mean over the l real rows
        const long long s = r / b.pool_rows;
        const int l = dib_set_len(b.set_sizes, s, b.pool_rows);
        if (r - s * b.pool_rows < l) dy = b.dy_pool[s * a.ld + e] * (1.f / (float)l);
      } else if (b.dy_pool) {
        dy = b.dy_pool[(r / b.pool_rows) * a.ld + e] * b.pool_scale;
      }
      for (int q = 0; q < 4; ++q)
        if (b.dy[q]) dy += b.dy[q][r * a.ld + e];
      dg[k] = fmaf(dy, xh[k], dg[k]);
      db[k] += dy;
      g[k] = dy * a.gamma[e];
      s1 += g[k];
      s2 = fmaf(g[k], xh[k], s2);
    }
    const float m1 = dib_warp_sum(s1) / (float)E, m2 = dib_warp_sum(s2) / (float)E;
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const int e = lane + 32 * k;
      if (e >= a.ld) continue;
      const float dz = e < E ? rstd * (g[k] - m1 - xh[k] * m2) : 0.f;
      b.d_res[r * a.ld + e] = dib_maybe_round(dz, a.round_out);
      if (b.d_branch)
        b.d_branch[r * a.ld + e] = e < E ? dib_maybe_round(dz * dib_act_grad(b.branch_act, a.b[r * a.ld + e], b.alpha), a.round_out) : 0.f;
    }
  }
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    const int e = lane + 32 * k;
    if (e < 128) { red[warp][0][e] = dg[k]; red[warp][1][e] = db[k]; }
  }
  __syncthreads();
  float* part = b.part + (long long)blockIdx.x * b.split_stride;
  for (int e = threadIdx.x; e < E; e += kLnWarps * 32) {
    float sg = 0.f, sb = 0.f;
    for (int w = 0; w < kLnWarps; ++w) { sg += red[w][0][e]; sb += red[w][1][e]; }
    part[b.gamma_off + e] = sg;
    part[b.beta_off + e] = sb;
  }
}

// pooled[s, e] = (sum_p x[s L + p, e]) / L, and its reverse d x[s L + p, e] = d pooled[s, e] / L lives in ln_bwd_kernel
__global__ void pool_fwd_kernel(const float* x, int ld, int E, int L, long long sets, float* out, int ldo, int round_out) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= sets * ldo) return;
  const long long s = i / ldo;
  const int e = (int)(i % ldo);
  float acc = 0.f;
  if (e < E)
    for (int p = 0; p < L; ++p) acc += x[(s * L + p) * ld + e];
  out[i] = e < E ? dib_maybe_round(acc / (float)L, round_out) : 0.f;
}

__global__ void sum_rows_kernel(DibSumRows a) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= a.count) return;
  float s = 0.f;
  for (int q = 0; q < 4; ++q)
    if (a.src[q]) s += a.src[q][i];
  a.dst[i] = s;
}

}  // namespace

size_t dib_attn_smem_bytes(int L, int dk, bool backward) {
  const size_t rows = (size_t)L * (dk + 1), sq = (size_t)L * (L + 1);
  return sizeof(float) * (backward ? 4 * rows + 2 * sq + L : 3 * rows + sq);
}

// the dynamic shared-memory opt-in of both attention kernels at their largest shape (L = 64, dk = 128): a host call made
// once per model creation, outside any stream capture
cudaError_t dib_attn_prepare() {
  cudaError_t e = cudaFuncSetAttribute(attn_fwd_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                       (int)dib_attn_smem_bytes(64, 128, false));
  if (e != cudaSuccess) return e;
  return cudaFuncSetAttribute(attn_bwd_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)dib_attn_smem_bytes(64, 128, true));
}

cudaError_t dib_launch_attn_fwd(const DibAttnArgs& a, cudaStream_t st) {
  const size_t smem = dib_attn_smem_bytes(a.L, a.dk, false);
  if (a.sets == 0) return cudaSuccess;
  attn_fwd_kernel<<<dim3(a.heads, (unsigned)a.sets), kAttnThreads, smem, st>>>(a);
  dib_note_launch();
  return cudaGetLastError();
}

cudaError_t dib_launch_attn_bwd(const DibAttnArgs& a, cudaStream_t st) {
  const size_t smem = dib_attn_smem_bytes(a.L, a.dk, true);
  if (a.sets == 0) return cudaSuccess;
  attn_bwd_kernel<<<dim3(a.heads, (unsigned)a.sets), kAttnThreads, smem, st>>>(a);
  dib_note_launch();
  return cudaGetLastError();
}

cudaError_t dib_launch_ln_fwd(const DibLayerNorm& a, cudaStream_t st) {
  const unsigned grid = (unsigned)DIB_CEIL_DIV(a.rows, (long long)kLnWarps);
  if (grid == 0) return cudaSuccess;
  ln_fwd_kernel<<<grid, kLnWarps * 32, 0, st>>>(a);
  dib_note_launch();
  return cudaGetLastError();
}

cudaError_t dib_launch_ln_bwd(const DibLayerNorm& a, const DibLayerNormBwd& b, cudaStream_t st) {
  if (b.nsplit < 1) return cudaSuccess;
  ln_bwd_kernel<<<b.nsplit, kLnWarps * 32, 0, st>>>(a, b);
  dib_note_launch();
  return cudaGetLastError();
}

cudaError_t dib_launch_pool_fwd(const float* x, int ld, int E, int L, int64_t sets, float* out, int ldo, int round_out,
                                cudaStream_t st) {
  const long long count = sets * ldo;
  if (count == 0) return cudaSuccess;
  pool_fwd_kernel<<<(unsigned)DIB_CEIL_DIV(count, 256ll), 256, 0, st>>>(x, ld, E, L, sets, out, ldo, round_out);
  dib_note_launch();
  return cudaGetLastError();
}

cudaError_t dib_launch_sum_rows(const DibSumRows& a, cudaStream_t st) {
  if (a.count == 0) return cudaSuccess;
  sum_rows_kernel<<<(unsigned)DIB_CEIL_DIV(a.count, 256ll), 256, 0, st>>>(a);
  dib_note_launch();
  return cudaGetLastError();
}
