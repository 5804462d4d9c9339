// NEXT ROW f3 (SURVEY.md section 8f): the InfoNCE head of the reference's custom training loop.
//   utils.get_scaled_similarity  (utils.py:127-175, pairwise distances utils.py:75-125)
//   loss_infonce = mean_i CE(i, S[i,:]) + mean_i CE(i, S^T[i,:])   (train.py:203-213)
// and the reverse mode GradientTape takes through both (train.py:216-219).  The [n, n] similarity matrix is
// written once; row/column log-sum-exps, the loss and both embedding gradients are read back from it, all
// reductions in a fixed order (deterministic).  CUDA-core fp32: n <= a few thousand, d <= 512 -- the work is
// O(n^2 d) elementwise, not a contraction worth a tensor-core path except for 'cosine'/'l2sq', which the
// reference itself expresses as a matmul; they share this kernel for one code path and bit-stable results.
#include "dib_common.cuh"
#include "dib_kernels.h"

namespace {

enum { SIM_L2SQ = 0, SIM_L2 = 1, SIM_L1 = 2, SIM_LINF = 3, SIM_COS = 4 };
constexpr float kL2Eps = 1e-9f;            // utils.py:150
constexpr int kGradThreads = 128, kMaxDimPerThread = 4;   // d <= 512

__device__ __forceinline__ float signf(float v) { return (v > 0.f) - (v < 0.f); }

// tile of 8 rows (e1) x 32 rows (e2) per block, d walked in chunks of 32 through shared memory
__global__ void __launch_bounds__(256)
dib_similarity_kernel(int kind, const float* __restrict__ e1, long long n, const float* __restrict__ e2, long long m, int d,
                      float inv_t, float* __restrict__ out) {
  __shared__ float sa[8][32], sbt[32][33];
  const int tj = threadIdx.x & 31, ti = threadIdx.x >> 5;
  const long long i0 = (long long)blockIdx.y * 8, j0 = (long long)blockIdx.x * 32;
  float ss = 0.f, s1 = 0.f, mx = 0.f, dot = 0.f, na = 0.f, nb = 0.f;
  for (int k0 = 0; k0 < d; k0 += 32) {
    {
      const long long i = i0 + ti;
      sa[ti][tj] = (i < n && k0 + tj < d) ? e1[i * d + k0 + tj] : 0.f;
#pragma unroll
      for (int r = 0; r < 4; ++r) {
        const long long j = j0 + ti * 4 + r;
        sbt[ti * 4 + r][tj] = (j < m && k0 + tj < d) ? e2[j * d + k0 + tj] : 0.f;
      }
    }
    __syncthreads();
    const int kmax = min(32, d - k0);
    for (int k = 0; k < kmax; ++k) {
      const float a = sa[ti][k], b = sbt[tj][k], df = a - b;
      ss = fmaf(df, df, ss); s1 += fabsf(df); mx = fmaxf(mx, fabsf(df));
      dot = fmaf(a, b, dot); na = fmaf(a, a, na); nb = fmaf(b, b, nb);
    }
    __syncthreads();
  }
  const long long i = i0 + ti, j = j0 + tj;
  if (i >= n || j >= m) return;
  float s;
  switch (kind) {
    case SIM_L2SQ: s = -ss; break;
    case SIM_L2: s = -sqrtf(ss + kL2Eps); break;
    case SIM_L1: s = -s1; break;
    case SIM_LINF: s = -mx; break;
    default: s = dot / (sqrtf(na) * sqrtf(nb)); break;
  }
  out[i * m + j] = s * inv_t;
}

// lse[0..n): log sum_j exp S[i,j] (one warp per row);  lse[n..2n): log sum_i exp S[i,j] (32 columns x 8 row groups)
__global__ void __launch_bounds__(256)
dib_infonce_row_lse_kernel(const float* __restrict__ S, int n, float* __restrict__ lse) {
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int i = blockIdx.x * 8 + warp;
  if (i >= n) return;
  const float* row = S + (long long)i * n;
  float mxv = -INFINITY;
  for (int j = lane; j < n; j += 32) mxv = fmaxf(mxv, row[j]);
  for (int o = 16; o; o >>= 1) mxv = fmaxf(mxv, __shfl_xor_sync(0xffffffffu, mxv, o));
  float s = 0.f;
  for (int j = lane; j < n; j += 32) s += expf(row[j] - mxv);
  s = dib_warp_sum(s);
  if (lane == 0) lse[i] = mxv + logf(s);
}

__global__ void __launch_bounds__(256)
dib_infonce_col_lse_kernel(const float* __restrict__ S, int n, float* __restrict__ lse) {
  __shared__ float smx[8][32], ssum[8][32];
  const int tj = threadIdx.x & 31, tg = threadIdx.x >> 5;
  const int j = blockIdx.x * 32 + tj;
  float mxv = -INFINITY;
  if (j < n) for (int i = tg; i < n; i += 8) mxv = fmaxf(mxv, S[(long long)i * n + j]);
  smx[tg][tj] = mxv;
  __syncthreads();
  float cm = smx[0][tj];
#pragma unroll
  for (int g = 1; g < 8; ++g) cm = fmaxf(cm, smx[g][tj]);
  float s = 0.f;
  if (j < n) for (int i = tg; i < n; i += 8) s += expf(S[(long long)i * n + j] - cm);
  ssum[tg][tj] = s;
  __syncthreads();
  if (tg == 0 && j < n) {
    float t = 0.f;
#pragma unroll
    for (int g = 0; g < 8; ++g) t += ssum[g][tj];
    lse[n + j] = cm + logf(t);
  }
}

// aux[0..n) = |e1_i|, aux[n..2n) = |e2_j| (cosine only); one warp per row of either matrix
__global__ void __launch_bounds__(256)
dib_row_norm_kernel(const float* __restrict__ e1, const float* __restrict__ e2, int n, int d, float* __restrict__ aux) {
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int r = blockIdx.x * 8 + warp;
  if (r >= 2 * n) return;
  const float* p = (r < n ? e1 + (long long)r * d : e2 + (long long)(r - n) * d);
  float s = 0.f;
  for (int k = lane; k < d; k += 32) s = fmaf(p[k], p[k], s);
  s = dib_warp_sum(s);
  if (lane == 0) aux[r] = sqrtf(s);
}

__global__ void __launch_bounds__(256)
dib_infonce_loss_kernel(const float* __restrict__ S, const float* __restrict__ lse, int n, float* __restrict__ out_loss) {
  __shared__ float red[8];
  float v = 0.f;
  for (int i = threadIdx.x; i < n; i += 256) v += lse[i] + lse[n + i] - 2.f * S[(long long)i * n + i];
  v = dib_warp_sum(v);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
  __syncthreads();
  if (threadIdx.x == 0) {
    float t = 0.f;
    for (int w = 0; w < 8; ++w) t += red[w];
    out_loss[0] = t / (float)n;
  }
}

// d loss / d (row r of `self`), self = e1 (TRANSPOSED = false) or e2 (true); `other` is the opposite matrix.
//   dS_ij = [softmax_row(S)_ij + softmax_col(S)_ij - 2 delta_ij] / n ;  d self_r = sum_o dS * d s / d self_r
template <bool TRANSPOSED>
__global__ void __launch_bounds__(kGradThreads)
dib_infonce_grad_kernel(int kind, const float* __restrict__ self, const float* __restrict__ other, int n, int d, float inv_t,
                        const float* __restrict__ S, const float* __restrict__ lse, const float* __restrict__ norms,
                        float* __restrict__ d_self) {
  extern __shared__ float sm[];
  float* a = sm;                         // [d] this row
  float* w = sm + d;                     // [kGradThreads] dS for the chunk
  float* ex = w + kGradThreads;          // [kGradThreads] per-pair extra (l2: 1/dist, cosine: c, linf: max_k |a_k - b_k|)
  const int r = blockIdx.x, tid = threadIdx.x;
  for (int k = tid; k < d; k += kGradThreads) a[k] = self[(long long)r * d + k];
  const float lse_r = lse[TRANSPOSED ? n + r : r];
  const float* lse_o = lse + (TRANSPOSED ? 0 : n);
  const float inv_na = kind == SIM_COS ? 1.f / norms[TRANSPOSED ? n + r : r] : 0.f;
  const float* norm_o = norms + (TRANSPOSED ? 0 : n);
  float acc[kMaxDimPerThread];
#pragma unroll
  for (int u = 0; u < kMaxDimPerThread; ++u) acc[u] = 0.f;
  __syncthreads();
  for (int o0 = 0; o0 < n; o0 += kGradThreads) {
    const int o = o0 + tid;
    if (o < n) {
      const float s = TRANSPOSED ? S[(long long)o * n + r] : S[(long long)r * n + o];
      w[tid] = (expf(s - lse_r) + expf(s - lse_o[o]) - (o == r ? 2.f : 0.f)) / (float)n;
      float e = 0.f;
      if (kind == SIM_L2) e = 1.f / (-s / inv_t);                 // sqrt(d2 + eps) = -S T
      else if (kind == SIM_COS) e = s / inv_t;                    // cos(a, b) = S T
      else if (kind == SIM_LINF) {              // the gradient is split evenly between tied maxima (TF _MinOrMaxGrad)
        const float* b = other + (long long)o * d;
        float best = -1.f; int ties = 0;
        for (int k = 0; k < d; ++k) {
          const float v = fabsf(a[k] - b[k]);
          if (v > best) { best = v; ties = 1; }
          else if (v == best) ++ties;
        }
        e = best;
        w[tid] *= 1.f / (float)ties;             // unchanged for one maximum
      }
      ex[tid] = e;
    }
    __syncthreads();
    const int cnt = min(kGradThreads, n - o0);
#pragma unroll
    for (int u = 0; u < kMaxDimPerThread; ++u) {
      const int k = tid + u * kGradThreads;
      if (k < d) {
        const float ak = a[k];
        float t = 0.f;
        for (int q = 0; q < cnt; ++q) {
          const float bk = other[(long long)(o0 + q) * d + k];
          const float df = ak - bk, wq = w[q];
          switch (kind) {
            case SIM_L2SQ: t = fmaf(wq, -2.f * df, t); break;
            case SIM_L2: t = fmaf(wq * ex[q], -df, t); break;
            case SIM_L1: t = fmaf(wq, -signf(df), t); break;
            case SIM_LINF: if (fabsf(df) == ex[q]) t = fmaf(wq, -signf(df), t); break;
            default: t = fmaf(wq, (bk / norm_o[o0 + q] - ex[q] * ak * inv_na) * inv_na, t); break;
          }
        }
        acc[u] += t;
      }
    }
    __syncthreads();
  }
#pragma unroll
  for (int u = 0; u < kMaxDimPerThread; ++u) {
    const int k = tid + u * kGradThreads;
    if (k < d) d_self[(long long)r * d + k] = acc[u] * inv_t;
  }
}

}  // namespace

cudaError_t dib_launch_similarity(int kind, const float* e1, int64_t n, const float* e2, int64_t m, int d, float temperature,
                                  float* out, cudaStream_t st) {
  if (n <= 0 || m <= 0) return cudaSuccess;
  dim3 grid((unsigned)DIB_CEIL_DIV(m, 32ll), (unsigned)DIB_CEIL_DIV(n, 8ll));
  dib_similarity_kernel<<<grid, 256, 0, st>>>(kind, e1, n, e2, m, d, 1.f / temperature, out);
  dib_note_launch();
  return cudaGetLastError();
}

// scratch: [n*n similarity | 2n log-sum-exps | 2n row norms]
cudaError_t dib_launch_infonce_head(int kind, const float* e1, const float* e2, int64_t n64, int d, float temperature,
                                    float* scratch, float* out_loss, float* d_e1, float* d_e2, cudaStream_t st) {
  const int n = (int)n64;
  if (n <= 0) return cudaSuccess;
  float* S = scratch;
  float* lse = scratch + (long long)n * n;
  float* norms = lse + 2 * n;
  const float inv_t = 1.f / temperature;
  cudaError_t e = dib_launch_similarity(kind, e1, n, e2, n, d, temperature, S, st);
  if (e != cudaSuccess) return e;
  dib_infonce_row_lse_kernel<<<DIB_CEIL_DIV(n, 8), 256, 0, st>>>(S, n, lse);
  dib_infonce_col_lse_kernel<<<DIB_CEIL_DIV(n, 32), 256, 0, st>>>(S, n, lse);
  dib_infonce_loss_kernel<<<1, 256, 0, st>>>(S, lse, n, out_loss);
  dib_note_launch(3);
  if (d_e1 || d_e2) {
    if (kind == SIM_COS) {
      dib_row_norm_kernel<<<DIB_CEIL_DIV(2 * n, 8), 256, 0, st>>>(e1, e2, n, d, norms);
      dib_note_launch();
    }
    const size_t smem = sizeof(float) * ((size_t)d + 2 * kGradThreads);
    if (d_e1) { dib_infonce_grad_kernel<false><<<n, kGradThreads, smem, st>>>(kind, e1, e2, n, d, inv_t, S, lse, norms, d_e1); dib_note_launch(); }
    if (d_e2) { dib_infonce_grad_kernel<true><<<n, kGradThreads, smem, st>>>(kind, e2, e1, n, d, inv_t, S, lse, norms, d_e2); dib_note_launch(); }
  }
  return cudaGetLastError();
}
