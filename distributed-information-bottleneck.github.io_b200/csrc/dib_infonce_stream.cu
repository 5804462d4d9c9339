// The InfoNCE loss of the reference's custom training loop (train.py:203-219) with memory linear in the batch:
//   S = get_scaled_similarity(e1, e2) = sim(e1_i, e2_j) / T           (utils.py:127-175)
//   loss = mean_i CE(i, S[i,:]) + mean_i CE(i, S^T[i,:])
//   d e1_i = sum_j w_ij d s_ij / d e1_i,  d e2_j = sum_i w_ij d s_ij / d e2_j,
//   w_ij = (exp(s_ij - r_i) + exp(s_ij - c_j) - 2 delta_ij) / n,  r = row log-sum-exp, c = column log-sum-exp.
// S is never stored: every sweep recomputes its 32 x 32 tiles from e1 / e2 rows staged in shared memory.
//   1. row sweep    (self = e1, other = e2): r_i by an online max / sum, and the diagonal s_ii;
//   2. column sweep (self = e2, other = e1): c_j -- every similarity kind is symmetric bit for bit
//      (a - b = -(b - a), fmaf(a, b) = fmaf(b, a)), so the column sweep is the row sweep with the operands swapped;
//   3. loss: sum_i (r_i + c_i - 2 s_ii) in a fixed order (= n * loss, the stats slot);
//   4. gradient sweeps, again once per side with the roles swapped.
// Arithmetic is fp32 on CUDA cores in the difference form of dib_similarity_kernel (dib_infonce.cu): every s_ij is
// accumulated over d in the same order, so it equals the value that kernel writes.  Nothing is accumulated with atomics:
// every sum has a fixed order, so results are bit-identical run to run and under graph replay.  d <= 512.
#include "dib_common.cuh"
#include "dib_kernels.h"

namespace {

enum { SIM_L2SQ = 0, SIM_L2 = 1, SIM_L1 = 2, SIM_LINF = 3, SIM_COS = 4 };
constexpr float kL2Eps = 1e-9f;          // utils.py:150
constexpr int kTile = 32;                // rows of `self` per block, rows of `other` per tile
constexpr int kThreads = 256;            // 8 warps x 4 rows each; lane = column of the tile
constexpr int kRowsPerWarp = kTile / (kThreads / 32);

__host__ __device__ constexpr int smem_ld(int d) { return d | 1; }     // odd row stride: column walks are conflict-free

// `rows` rows of m [*, d] (leading dimension ldm) from row r0 into s[rows][ld]; rows past n are zero.  With COS, nrm[r] is
// |row| accumulated over d in order (the per-pair na / nb of dib_similarity_kernel, which depend on one row only).
template <int KIND>
__device__ __forceinline__ void stage_rows(const float* __restrict__ m, int ldm, long long n, long long r0, int d, float* s,
                                           float* nrm) {
  const int ld = smem_ld(d);
  for (int idx = threadIdx.x; idx < kTile * d; idx += kThreads) {
    const int r = idx / d, k = idx - r * d;
    const long long row = r0 + r;
    s[r * ld + k] = row < n ? m[row * ldm + k] : 0.f;
  }
  if (KIND == SIM_COS) {
    __syncthreads();
    if (threadIdx.x < kTile) {
      const float* p = s + threadIdx.x * ld;
      float q = 0.f;
      for (int k = 0; k < d; ++k) q = fmaf(p[k], p[k], q);
      nrm[threadIdx.x] = sqrtf(q);
    }
  }
}

// the similarities of rows (i0 .. i0+3) of sa with row j of sb, scaled by inv_t; am[] = argmax_k |a_k - b_k| (LINF)
template <int KIND>
__device__ __forceinline__ void tile_similarity(const float* sa, int i0, const float* sb, int j, int d, const float* na,
                                                const float* nb, float inv_t, float (&s)[kRowsPerWarp], int (&am)[kRowsPerWarp]) {
  const int ld = smem_ld(d);
  float acc[kRowsPerWarp];
#pragma unroll
  for (int r = 0; r < kRowsPerWarp; ++r) { acc[r] = 0.f; am[r] = 0; }
  const float* b = sb + j * ld;
  for (int k = 0; k < d; ++k) {
    const float bk = b[k];
#pragma unroll
    for (int r = 0; r < kRowsPerWarp; ++r) {
      const float a = sa[(i0 + r) * ld + k];
      if (KIND == SIM_L2SQ || KIND == SIM_L2) { const float df = a - bk; acc[r] = fmaf(df, df, acc[r]); }
      else if (KIND == SIM_L1) acc[r] += fabsf(a - bk);
      else if (KIND == SIM_LINF) { const float v = fabsf(a - bk); if (v > acc[r]) { acc[r] = v; am[r] = k; } }
      else acc[r] = fmaf(a, bk, acc[r]);
    }
  }
#pragma unroll
  for (int r = 0; r < kRowsPerWarp; ++r) {
    float v;
    if (KIND == SIM_L2SQ) v = -acc[r];
    else if (KIND == SIM_L2) v = -sqrtf(acc[r] + kL2Eps);
    else if (KIND == SIM_L1 || KIND == SIM_LINF) v = -acc[r];
    else v = acc[r] / (na[i0 + r] * nb[j]);
    s[r] = v * inv_t;
  }
}

// lse[i] = log sum_j exp S(self_i, other_j) over all n rows of `other`; diag[i] = S(self_i, other_i) when diag != nullptr.
// One block per 32 rows of `self`; each lane keeps an online (max, sum) over the columns j = lane (mod 32), merged across
// the warp in a fixed tree at the end.
template <int KIND>
__global__ void __launch_bounds__(kThreads)
dib_infonce_lse_kernel(const float* __restrict__ self, int ld_self, const float* __restrict__ other, int ld_other, int n, int d,
                       float inv_t, float* __restrict__ lse, float* __restrict__ diag) {
  extern __shared__ float sm[];
  const int ld = smem_ld(d);
  float* sa = sm;
  float* sb = sa + kTile * ld;
  float* na = sb + kTile * ld;
  float* nb = na + kTile;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, i0 = warp * kRowsPerWarp;
  const long long row0 = (long long)blockIdx.x * kTile;
  stage_rows<KIND>(self, ld_self, n, row0, d, sa, na);
  float mx[kRowsPerWarp], sum[kRowsPerWarp];
#pragma unroll
  for (int r = 0; r < kRowsPerWarp; ++r) { mx[r] = -INFINITY; sum[r] = 0.f; }
  for (int j0 = 0; j0 < n; j0 += kTile) {
    __syncthreads();
    stage_rows<KIND>(other, ld_other, n, j0, d, sb, nb);
    __syncthreads();
    const int j = j0 + lane;
    if (j >= n) continue;
    float s[kRowsPerWarp]; int am[kRowsPerWarp];
    tile_similarity<KIND>(sa, i0, sb, lane, d, na, nb, inv_t, s, am);
#pragma unroll
    for (int r = 0; r < kRowsPerWarp; ++r) {
      if (s[r] > mx[r]) { sum[r] = sum[r] * expf(mx[r] - s[r]) + 1.f; mx[r] = s[r]; }
      else sum[r] += expf(s[r] - mx[r]);
      if (diag && row0 + i0 + r == j) diag[j] = s[r];
    }
  }
#pragma unroll
  for (int r = 0; r < kRowsPerWarp; ++r) {
    float m = mx[r], t = sum[r];
    for (int o = 16; o; o >>= 1) {
      const float m2 = __shfl_down_sync(0xffffffffu, m, o), t2 = __shfl_down_sync(0xffffffffu, t, o);
      if (m2 == -INFINITY) continue;                       // that lane saw no column
      if (m == -INFINITY) { m = m2; t = t2; continue; }
      const float mm = fmaxf(m, m2);
      t = t * expf(m - mm) + t2 * expf(m2 - mm);
      m = mm;
    }
    const long long i = row0 + i0 + r;
    if (lane == 0 && i < n) lse[i] = m + logf(t);
  }
}

// out[0] = sum_i (r_i + c_i - 2 s_ii) (= n * loss) and out_acc[0] = 0, one block, fixed order
__global__ void __launch_bounds__(kThreads)
dib_infonce_stream_loss_kernel(const float* __restrict__ r, const float* __restrict__ c, const float* __restrict__ diag, int n,
                               float* __restrict__ out, float* __restrict__ out_acc) {
  __shared__ float red[kThreads / 32];
  float v = 0.f;
  for (int i = threadIdx.x; i < n; i += kThreads) v += r[i] + c[i] - 2.f * diag[i];
  v = dib_warp_sum(v);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
  __syncthreads();
  if (threadIdx.x == 0) {
    float t = 0.f;
    for (int w = 0; w < kThreads / 32; ++w) t += red[w];
    out[0] = t;
    if (out_acc) out_acc[0] = 0.f;
  }
}

// d self_i = sum_o w_io d s_io / d self_i, w_io = (exp(s_io - lse_self_i) + exp(s_io - lse_other_o) - 2 delta_io) / n, with
// s_io = S(self_i, other_o).  One block per 32 rows of `self`; per tile the weights and the per-pair factor go to shared
// memory, then every thread adds the tile's contribution to its own (row, dim) elements of the accumulator.  Output rows are
// written with leading dimension ld_out (pad columns zeroed) and rounded to TF32 when round_out.
template <int KIND>
__global__ void __launch_bounds__(kThreads)
dib_infonce_grad_stream_kernel(const float* __restrict__ self, int ld_self, const float* __restrict__ other, int ld_other, int n,
                               int d, float inv_t, const float* __restrict__ lse_self, const float* __restrict__ lse_other,
                               float* __restrict__ d_self, int ld_out, int round_out) {
  extern __shared__ float sm[];
  const int ld = smem_ld(d);
  float* sa = sm;
  float* sb = sa + kTile * ld;
  float* acc = sb + kTile * ld;                       // [kTile][d]
  float* wt = acc + kTile * d;                        // [kTile][kTile + 1]
  float* ex = wt + kTile * (kTile + 1);               // [kTile][kTile + 1]: l2 1/distance, cosine cos, linf argmax bits
  float* na = ex + kTile * (kTile + 1);
  float* nb = na + kTile;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, i0 = warp * kRowsPerWarp;
  const long long row0 = (long long)blockIdx.x * kTile;
  const float inv_n = 1.f / (float)n;
  stage_rows<KIND>(self, ld_self, n, row0, d, sa, na);
  for (int idx = threadIdx.x; idx < kTile * d; idx += kThreads) acc[idx] = 0.f;
  float lr[kRowsPerWarp];
#pragma unroll
  for (int r = 0; r < kRowsPerWarp; ++r) lr[r] = row0 + i0 + r < n ? lse_self[row0 + i0 + r] : 0.f;
  for (int j0 = 0; j0 < n; j0 += kTile) {
    __syncthreads();
    stage_rows<KIND>(other, ld_other, n, j0, d, sb, nb);
    __syncthreads();
    {
      const int j = j0 + lane;
      float s[kRowsPerWarp]; int am[kRowsPerWarp];
      tile_similarity<KIND>(sa, i0, sb, lane, d, na, nb, inv_t, s, am);
      const float lo = j < n ? lse_other[j] : 0.f;
#pragma unroll
      for (int r = 0; r < kRowsPerWarp; ++r) {
        const long long i = row0 + i0 + r;
        float w = 0.f, e = 0.f;
        if (i < n && j < n) {
          w = (expf(s[r] - lr[r]) + expf(s[r] - lo) - (i == j ? 2.f : 0.f)) * inv_n;
          if (KIND == SIM_L2) e = 1.f / (-s[r] / inv_t);        // sqrt(d2 + eps) = -S T
          else if (KIND == SIM_COS) e = s[r] / inv_t;           // cos(a, b) = S T
          else if (KIND == SIM_LINF) e = __int_as_float(am[r]);
        }
        wt[(i0 + r) * (kTile + 1) + lane] = w;
        ex[(i0 + r) * (kTile + 1) + lane] = e;
      }
    }
    __syncthreads();
    const int cnt = min(kTile, n - j0);
#pragma unroll
    for (int r = 0; r < kRowsPerWarp; ++r) {
      const int il = i0 + r;
      const float* wr = wt + il * (kTile + 1);
      const float* er = ex + il * (kTile + 1);
      const float inv_na = KIND == SIM_COS ? 1.f / na[il] : 0.f;
      for (int k = lane; k < d; k += 32) {
        const float ak = sa[il * ld + k];
        float t = 0.f;
        for (int q = 0; q < cnt; ++q) {
          const float bk = sb[q * ld + k], df = ak - bk, wq = wr[q];
          if (KIND == SIM_L2SQ) t = fmaf(wq, -2.f * df, t);
          else if (KIND == SIM_L2) t = fmaf(wq * er[q], -df, t);
          else if (KIND == SIM_L1) t = fmaf(wq, -((df > 0.f) - (df < 0.f)), t);
          else if (KIND == SIM_LINF) { if (__float_as_int(er[q]) == k) t = fmaf(wq, -(float)((df > 0.f) - (df < 0.f)), t); }
          else t = fmaf(wq, (bk / nb[q] - er[q] * ak * inv_na) * inv_na, t);
        }
        acc[il * d + k] += t;
      }
    }
  }
  __syncthreads();
#pragma unroll
  for (int r = 0; r < kRowsPerWarp; ++r) {
    const long long i = row0 + i0 + r;
    if (i >= n) continue;
    for (int k = lane; k < ld_out; k += 32)
      d_self[i * ld_out + k] = k < d ? dib_maybe_round(acc[(i0 + r) * d + k] * inv_t, round_out) : 0.f;
  }
}

size_t lse_smem(int d) { return sizeof(float) * (2 * (size_t)kTile * smem_ld(d) + 2 * kTile); }
size_t grad_smem(int d) {
  return sizeof(float) * (2 * (size_t)kTile * smem_ld(d) + (size_t)kTile * d + 2 * kTile * (kTile + 1) + 2 * kTile);
}

template <int KIND>
cudaError_t launch_loss(const DibInfonceStream& a, cudaStream_t st) {
  const int n = (int)a.n, d = a.d;
  const size_t smem = lse_smem(d);
  cudaError_t e = cudaFuncSetAttribute(dib_infonce_lse_kernel<KIND>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  if (e != cudaSuccess) return e;
  const unsigned blocks = (unsigned)DIB_CEIL_DIV(n, kTile);
  float *r = a.scratch, *c = a.scratch + n, *diag = a.scratch + 2 * (long long)n;
  dib_infonce_lse_kernel<KIND><<<blocks, kThreads, smem, st>>>(a.e1, a.ld1, a.e2, a.ld2, n, d, 1.f / a.temperature, r, diag);
  dib_infonce_lse_kernel<KIND><<<blocks, kThreads, smem, st>>>(a.e2, a.ld2, a.e1, a.ld1, n, d, 1.f / a.temperature, c, nullptr);
  dib_infonce_stream_loss_kernel<<<1, kThreads, 0, st>>>(r, c, diag, n, a.loss_sum, a.acc_zero);
  dib_note_launch(3);
  return cudaGetLastError();
}

template <int KIND>
cudaError_t launch_grads(const DibInfonceStream& a, cudaStream_t st) {
  const int n = (int)a.n, d = a.d;
  const size_t smem = grad_smem(d);
  cudaError_t e = cudaFuncSetAttribute(dib_infonce_grad_stream_kernel<KIND>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  if (e != cudaSuccess) return e;
  const unsigned blocks = (unsigned)DIB_CEIL_DIV(n, kTile);
  const float *r = a.scratch, *c = a.scratch + n;
  if (a.d_e1) {
    dib_infonce_grad_stream_kernel<KIND><<<blocks, kThreads, smem, st>>>(a.e1, a.ld1, a.e2, a.ld2, n, d, 1.f / a.temperature, r,
                                                                         c, a.d_e1, a.ld_d1, a.round_out);
    dib_note_launch();
  }
  if (a.d_e2) {
    dib_infonce_grad_stream_kernel<KIND><<<blocks, kThreads, smem, st>>>(a.e2, a.ld2, a.e1, a.ld1, n, d, 1.f / a.temperature, c,
                                                                         r, a.d_e2, a.ld_d2, a.round_out);
    dib_note_launch();
  }
  return cudaGetLastError();
}

}  // namespace

cudaError_t dib_launch_infonce_stream_loss(const DibInfonceStream& a, cudaStream_t st) {
  if (a.n <= 0) return cudaSuccess;
  switch (a.kind) {
    case SIM_L2SQ: return launch_loss<SIM_L2SQ>(a, st);
    case SIM_L2: return launch_loss<SIM_L2>(a, st);
    case SIM_L1: return launch_loss<SIM_L1>(a, st);
    case SIM_LINF: return launch_loss<SIM_LINF>(a, st);
    default: return launch_loss<SIM_COS>(a, st);
  }
}

cudaError_t dib_launch_infonce_stream_grads(const DibInfonceStream& a, cudaStream_t st) {
  if (a.n <= 0) return cudaSuccess;
  switch (a.kind) {
    case SIM_L2SQ: return launch_grads<SIM_L2SQ>(a, st);
    case SIM_L2: return launch_grads<SIM_L2>(a, st);
    case SIM_L1: return launch_grads<SIM_L1>(a, st);
    case SIM_LINF: return launch_grads<SIM_LINF>(a, st);
    default: return launch_grads<SIM_COS>(a, st);
  }
}
