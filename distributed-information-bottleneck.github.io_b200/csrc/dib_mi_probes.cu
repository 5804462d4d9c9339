// dib_mi_probes.cu -- per-probe information maps (nb-particle cell 8, :521-570): for M probe encodings and B batches of
// encoded data rows, the InfoNCE lower and leave-one-out upper bound of every probe, float64 throughout.
//
//   u_p      = mu_p + exp(lv_p / 2) eps_pb                                   (:554)
//   ls_p     = -1/2 sum_e eps_pbe^2 - 1/2 sum_e lv_pe + c                     (:557, (u - mu_p) / sigma_p = eps)
//   l_pj     = -1/2 sum_e (u_pe - mu_je)^2 exp(-lv_je) - 1/2 sum_e lv_je + c   (:563, j in batch b)
//   lower_pb = ls_p - [logsumexp(ls_p, l_p.) - log(N_b + 1)]                  (:566)
//   upper_pb = ls_p - [logsumexp(l_p.) - log N_b]                             (:569)
//   out[p]   = (mean_b lower_pb, mean_b upper_pb)
// with c = -E/2 log(2 pi).
//
// The quadratic form runs on the FP64 tensor pipe (mma.sync m16n8k4 .f64, sm_90) in the expanded form
//   q_pj + sum_e lv_je - 2c = [u'^2 | u' | 1] . [iv_j | -2 mu'_j iv_j | sum_e mu'^2_je iv_je + sum_e lv_je - 2c]
// where u' = u - s_b and mu' = mu - s_b are shifted by the batch's mean mu (s_b) to keep the cancellation of the expanded
// form small; the differences do not change.  K = 2E + 1, padded with zeros to a multiple of 4.
//
// Launches: (1) the batch shifts s_b, (2) the per-row table [R, Kp] in float64 (each data row converted once),
// (3) the main kernel, grid (ceil(M / 64), B): 4 warps x 16 probes, the batch's table rows streamed through a two-stage
// cp.async ring of 32 (E <= 64) or 16 rows, an online max / sum per probe, (per probe, batch) results to scratch, and
// (4) the mean over b in fixed order.  No atomics: repeated calls are bit-identical.
#include <cuda_runtime.h>
#include <math.h>
#include <stdint.h>

#include "dib_common.cuh"
#include "dib_kernels.h"

namespace {

constexpr int kPrTP = 64;                  // probes per block (4 warps x m16)
constexpr int kPrThreads = 128;
constexpr double kLog2Pi = 1.8378770664093454836;

__host__ __device__ inline int pr_kp(int E) { return (2 * E + 1 + 3) & ~3; }
// shared-memory row stride in doubles: = 4 (mod 8), so the 4 rows x 4 columns an m16n8k4 fragment load touches per half
// warp fall in distinct banks
__host__ __device__ inline int pr_stride(int E) { return ((pr_kp(E) + 7) & ~7) + 4; }

// s_b = the mean of mu over the rows of batch b (fixed-order block reduction); grid B, 256 threads
__global__ void __launch_bounds__(256)
dib_mi_probes_shift_kernel(const float* __restrict__ data, const long long* __restrict__ off, int E, double* __restrict__ shift) {
  __shared__ double red[8];
  const int b = blockIdx.x;
  const long long j0 = off[b], j1 = off[b + 1];
  for (int e = 0; e < E; ++e) {
    double s = 0.0;
    for (long long j = j0 + threadIdx.x; j < j1; j += blockDim.x) s += (double)data[j * 2 * E + e];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = s;
    __syncthreads();
    if (threadIdx.x == 0) {
      double t = 0.0;
      for (int w = 0; w < 8; ++w) t += red[w];
      shift[(long long)b * E + e] = j1 > j0 ? t / (double)(j1 - j0) : 0.0;
    }
    __syncthreads();
  }
}

// table row j of batch b: [iv (E) | -2 mu' iv (E) | sum mu'^2 iv + sum lv - 2c | 0 pad]; grid (chunks, B), one thread per row
__global__ void __launch_bounds__(256)
dib_mi_probes_table_kernel(const float* __restrict__ data, const long long* __restrict__ off, int E,
                           const double* __restrict__ shift, double* __restrict__ table) {
  const int b = blockIdx.y, Kp = pr_kp(E);
  const long long j1 = off[b + 1];
  const double* sb = shift + (long long)b * E;
  const double c2 = (double)E * kLog2Pi;                    // -2c
  for (long long j = off[b] + (long long)blockIdx.x * blockDim.x + threadIdx.x; j < j1; j += (long long)gridDim.x * blockDim.x) {
    const float* r = data + j * 2 * E;
    double* t = table + j * Kp;
    double last = c2;
    for (int e = 0; e < E; ++e) {
      const double lv = (double)r[E + e], iv = exp(-lv), mu = (double)r[e] - sb[e];
      t[e] = iv;
      t[E + e] = -2.0 * mu * iv;
      last += mu * mu * iv + lv;
    }
    t[2 * E] = last;
    for (int k = 2 * E + 1; k < Kp; ++k) t[k] = 0.0;
  }
}

__device__ __forceinline__ void pr_dmma(double (&d)[4], double a0, double a1, double b0) {
  asm volatile("mma.sync.aligned.m16n8k4.row.col.f64.f64.f64.f64 {%0, %1, %2, %3}, {%4, %5}, {%6}, {%0, %1, %2, %3};"
               : "+d"(d[0]), "+d"(d[1]), "+d"(d[2]), "+d"(d[3])
               : "d"(a0), "d"(a1), "d"(b0));
}

__device__ __forceinline__ void pr_cp_async16(void* smem, const void* gmem, int bytes) {
  const unsigned s = (unsigned)__cvta_generic_to_shared(smem);
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(s), "l"(gmem), "r"(bytes));
}

// online log-sum-exp over one row's values of a tile: the rescale costs one exp per tile, not per value
template <int V>
__device__ __forceinline__ void pr_lse_add(double& m, double& s, const double (&l)[V], int valid) {
  double mx = -INFINITY;
#pragma unroll
  for (int k = 0; k < V; ++k) if (valid & (1 << k)) mx = fmax(mx, l[k]);
  if (mx == -INFINITY) return;
  if (mx > m) { s *= exp(m - mx); m = mx; }
#pragma unroll
  for (int k = 0; k < V; ++k) if (valid & (1 << k)) s += exp(l[k] - m);
}

__device__ __forceinline__ void pr_lse_merge(double& m, double& s, int lane_xor) {
  const double mo = __shfl_xor_sync(0xffffffffu, m, lane_xor), so = __shfl_xor_sync(0xffffffffu, s, lane_xor);
  const double mn = fmax(m, mo);
  if (mn == -INFINITY) return;
  s = s * exp(m - mn) + so * exp(mo - mn);
  m = mn;
}

template <int NT>
__global__ void __launch_bounds__(kPrThreads, 2)
dib_mi_probes_kernel(const float* __restrict__ probes, int M, int E, const double* __restrict__ table,
                     const long long* __restrict__ off, const double* __restrict__ shift, const float* __restrict__ eps,
                     unsigned long long seed, double* __restrict__ pb_out) {
  constexpr int TJ = NT * 8;
  extern __shared__ __align__(16) double sm[];
  const int Kp = pr_kp(E), S = pr_stride(E);
  double* sA = sm;                                  // [kPrTP][S]  (u'^2 | u' | 1 | 0)
  double* sB = sm + kPrTP * S;                      // [2][TJ][S]  table rows
  double* sLs = sB + 2 * TJ * S;                    // [kPrTP]     own log density
  const int b = blockIdx.y, tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, g = lane >> 2, t4 = lane & 3;
  const int p0 = blockIdx.x * kPrTP;
  const long long j0 = off[b], j1 = off[b + 1];
  const long long nb = j1 - j0;

  // stage the first data tile while the probe rows are built
  auto load_tile = [&](int stage, long long jt) {
    double* dst = sB + stage * TJ * S;
    const int chunks = Kp / 2;                      // 16-byte pieces per row
    for (int q = tid; q < TJ * chunks; q += kPrThreads) {
      const int r = q / chunks, c = q - r * chunks;
      const long long j = jt + r;
      const bool ok = j < j1;
      pr_cp_async16(dst + r * S + 2 * c, table + (ok ? j : j0) * Kp + 2 * c, ok ? 16 : 0);
    }
    asm volatile("cp.async.commit_group;" ::: "memory");
  };
  if (nb > 0) load_tile(0, j0);

  const double c = -0.5 * (double)E * kLog2Pi;
  if (tid < kPrTP) {
    const int p = p0 + tid;
    double* a = sA + tid * S;
    if (p < M) {
      const float* pr = probes + (long long)p * 2 * E;
      const double* sb = shift + (long long)b * E;
      double ls = c, e2 = 0.0;
      for (int e0 = 0; e0 < E; e0 += 4) {
        float nrm[4];
        if (!eps) dib_philox_normal4(seed, (uint32_t)b, (uint64_t)p, 0u, (uint32_t)(e0 >> 2), nrm);
        for (int k = 0; k < 4 && e0 + k < E; ++k) {
          const int e = e0 + k;
          const double z = eps ? (double)eps[((long long)b * M + p) * E + e] : (double)nrm[k];
          const double lv = (double)pr[E + e];
          const double u = (double)pr[e] + exp(0.5 * lv) * z - sb[e];
          a[e] = u * u;
          a[E + e] = u;
          e2 = fma(z, z, e2);
          ls -= 0.5 * lv;
        }
      }
      a[2 * E] = 1.0;
      sLs[tid] = ls - 0.5 * e2;
    } else {
      for (int k = 0; k <= 2 * E; ++k) a[k] = 0.0;
      sLs[tid] = 0.0;
    }
    for (int k = 2 * E + 1; k < Kp; ++k) a[k] = 0.0;
  }
  __syncthreads();

  // rows g and g + 8 of this warp's 16 probes
  double m_lo = -INFINITY, s_lo = 0.0, m_hi = -INFINITY, s_hi = 0.0;
  const double* aLo = sA + (warp * 16 + g) * S + t4;
  const double* aHi = aLo + 8 * S;
  int stage = 0;
  for (long long jt = j0; jt < j1; jt += TJ, stage ^= 1) {
    if (jt + TJ < j1) {
      load_tile(stage ^ 1, jt + TJ);
      asm volatile("cp.async.wait_group 1;" ::: "memory");
    } else {
      asm volatile("cp.async.wait_group 0;" ::: "memory");
    }
    __syncthreads();
    const double* bt = sB + stage * TJ * S + g * S + t4;
    double acc[NT][4];
#pragma unroll
    for (int n = 0; n < NT; ++n) acc[n][0] = acc[n][1] = acc[n][2] = acc[n][3] = 0.0;
    for (int k0 = 0; k0 < Kp; k0 += 4) {
      const double a0 = aLo[k0], a1 = aHi[k0];
#pragma unroll
      for (int n = 0; n < NT; ++n) pr_dmma(acc[n], a0, a1, bt[n * 8 * S + k0]);
    }
    // value (row, column n*8 + 2 t4 + i) = acc[n][i] (row g) / acc[n][2 + i] (row g + 8); l = -q / 2
    const long long left = j1 - jt;
    int valid = 0;
    double lo[2 * NT], hi[2 * NT];
#pragma unroll
    for (int n = 0; n < NT; ++n)
#pragma unroll
      for (int i = 0; i < 2; ++i) {
        if ((long long)(n * 8 + 2 * t4 + i) < left) valid |= 1 << (2 * n + i);
        lo[2 * n + i] = -0.5 * acc[n][i];
        hi[2 * n + i] = -0.5 * acc[n][2 + i];
      }
    pr_lse_add<2 * NT>(m_lo, s_lo, lo, valid);
    pr_lse_add<2 * NT>(m_hi, s_hi, hi, valid);
    __syncthreads();                               // this stage is refilled by the next iteration's load
  }
  pr_lse_merge(m_lo, s_lo, 1); pr_lse_merge(m_lo, s_lo, 2);
  pr_lse_merge(m_hi, s_hi, 1); pr_lse_merge(m_hi, s_hi, 2);
  if (t4 == 0) {
    const double ln1 = log((double)nb + 1.0), ln0 = log((double)nb);
#pragma unroll
    for (int r = 0; r < 2; ++r) {
      const int pl = warp * 16 + g + 8 * r, p = p0 + pl;
      if (p >= M) continue;
      const double ls = sLs[pl];
      const double lse = r ? m_hi + log(s_hi) : m_lo + log(s_lo);
      const double hiv = fmax(ls, lse), all = hiv + log1p(exp(-fabs(ls - lse)));
      double* o = pb_out + ((long long)b * M + p) * 2;
      if (nb < 1) { o[0] = o[1] = NAN; continue; }
      o[0] = ls - (all - ln1);                     // InfoNCE term       (:566)
      o[1] = ls - (lse - ln0);                     // leave-one-out term (:569)
    }
  }
}

// out[p] = the mean over b, in order b = 0 .. B-1
__global__ void __launch_bounds__(256)
dib_mi_probes_mean_kernel(const double* __restrict__ pb_out, int M, int B, double* __restrict__ out) {
  const long long p = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= M) return;
  double lo = 0.0, up = 0.0;
  for (int b = 0; b < B; ++b) { lo += pb_out[((long long)b * M + p) * 2]; up += pb_out[((long long)b * M + p) * 2 + 1]; }
  out[2 * p] = lo / B;
  out[2 * p + 1] = up / B;
}

size_t pr_align(size_t x) { return (x + 255) & ~(size_t)255; }

template <int NT>
size_t pr_smem(int E) { return (size_t)(kPrTP * pr_stride(E) + 2 * NT * 8 * pr_stride(E) + kPrTP) * sizeof(double); }

}  // namespace

// scratch: shifts [B, E] | per (batch, probe) results [B, m, 2] | row table [data_rows, Kp], the table last so that the
// launch needs no row count
size_t dib_mi_probes_scratch_bytes(int64_t m, int64_t data_rows, int B, int E) {
  return pr_align((size_t)B * E * sizeof(double)) + pr_align((size_t)B * m * 2 * sizeof(double)) +
         (size_t)data_rows * pr_kp(E) * sizeof(double);
}

cudaError_t dib_launch_mi_probes(const float* probes, int64_t m, const float* data, const int64_t* offsets, int B, int E,
                                 const float* eps, uint64_t seed, void* scratch, double* out, cudaStream_t st) {
  if (m <= 0 || B <= 0) return cudaSuccess;
  if (E < 1 || E > 128 || B > 65535) return cudaErrorInvalidValue;
  char* base = static_cast<char*>(scratch);
  double* shift = reinterpret_cast<double*>(base);
  double* pb = reinterpret_cast<double*>(base + pr_align((size_t)B * E * sizeof(double)));
  double* table = reinterpret_cast<double*>(reinterpret_cast<char*>(pb) + pr_align((size_t)B * m * 2 * sizeof(double)));
  const long long* off = reinterpret_cast<const long long*>(offsets);
  dib_mi_probes_shift_kernel<<<B, 256, 0, st>>>(data, off, E, shift);
  dib_note_launch();
  dib_mi_probes_table_kernel<<<dim3(64, B), 256, 0, st>>>(data, off, E, shift, table);
  dib_note_launch();
  const dim3 grid((unsigned)((m + kPrTP - 1) / kPrTP), B);
  if (E <= 64) {
    const size_t smem = pr_smem<4>(E);
    static bool attr = false;
    if (!attr) {
      cudaError_t e = cudaFuncSetAttribute(dib_mi_probes_kernel<4>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)pr_smem<4>(64));
      if (e != cudaSuccess) return e;
      attr = true;
    }
    dib_mi_probes_kernel<4><<<grid, kPrThreads, smem, st>>>(probes, (int)m, E, table, off, shift, eps, seed, pb);
  } else {
    const size_t smem = pr_smem<2>(E);
    static bool attr = false;
    if (!attr) {
      cudaError_t e = cudaFuncSetAttribute(dib_mi_probes_kernel<2>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)pr_smem<2>(128));
      if (e != cudaSuccess) return e;
      attr = true;
    }
    dib_mi_probes_kernel<2><<<grid, kPrThreads, smem, st>>>(probes, (int)m, E, table, off, shift, eps, seed, pb);
  }
  dib_note_launch();
  dib_mi_probes_mean_kernel<<<(unsigned)((m + 255) / 256), 256, 0, st>>>(pb, (int)m, B, out);
  dib_note_launch();
  return cudaGetLastError();
}
