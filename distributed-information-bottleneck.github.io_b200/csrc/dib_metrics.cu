// dib_metrics.cu -- compiled Keras metrics (dib_set_metrics): one launch after the compiled loss reduces the rows' output z,
// target y and sample weights into the metric tail of the statistics vector (layout: dib_metric_spec in dib_b200.h).
#include "dib_common.cuh"
#include "dib_kernels.h"

namespace {

constexpr int kThreads = 128;
constexpr int kWarps = kThreads / 32;
constexpr int kRowsPerThread = 4;          // rows per thread before the grid reaches kDibMetricMaxCtas

// Keras' AUC thresholds (metrics.AUC.__init__): [0 - epsilon] + [i / (T - 1) for i in 1 .. T-2] + [1 + epsilon], formed in
// Python doubles and stored as float32; the device doubles below are IEEE like Python's, so the float32 table is Keras'.
__device__ __forceinline__ float auc_threshold(int i, int T) {
  if (i == 0) return (float)(0.0 - 1e-7);
  if (i == T - 1) return (float)(1.0 + 1e-7);
  return (float)((double)i / (double)(T - 1));
}

// one row's mean metric m (averaged over the outputs, as Keras' MeanMetricWrapper functions reduce axis -1).  The libm
// expf / logf / log1pf (not the __expf intrinsics) throughout.
__device__ __forceinline__ float mean_metric(int kind, int from_logits, float threshold, const float* z, const float* y,
                                             long long row, int out_dim) {
  const float ep = 1e-7f;
  if (kind == DIB_METRIC_SPARSE_CATEGORICAL_ACCURACY || kind == DIB_METRIC_SPARSE_CATEGORICAL_CROSSENTROPY) {
    const float* zr = z + row * out_dim;
    const float t = y[row];
    if (kind == DIB_METRIC_SPARSE_CATEGORICAL_ACCURACY) {      // argmax (first maximum) == y, compared as floats
      float m = zr[0]; int am = 0;
      for (int j = 1; j < out_dim; ++j) if (zr[j] > m) { m = zr[j]; am = j; }
      return (float)am == t ? 1.f : 0.f;
    }
    const int label = dib_sparse_label(t, out_dim);
    if (label < 0) return __int_as_float(0x7fc00000);
    if (from_logits) {
      float m = zr[0];
      for (int j = 1; j < out_dim; ++j) m = fmaxf(m, zr[j]);
      float se = 0.f;
      for (int j = 0; j < out_dim; ++j) se += expf(zr[j] - m);
      return m + logf(se) - zr[label];
    }
    float se = 0.f;                                             // -log(p~_y / sum_j p~_j), p~ = clip(p, eps, 1 - eps)
    for (int j = 0; j < out_dim; ++j) se += fminf(fmaxf(zr[j], ep), 1.f - ep);
    return logf(se) - logf(fminf(fmaxf(zr[label], ep), 1.f - ep));
  }
  const float* zr = z + row * out_dim;
  const float* yr = y + row * out_dim;
  float s = 0.f;
  for (int j = 0; j < out_dim; ++j) {
    const float zz = zr[j], t = yr[j];
    float v;
    switch (kind) {
      case DIB_METRIC_MSE: { const float d = zz - t; v = d * d; break; }
      case DIB_METRIC_MAE: v = fabsf(zz - t); break;
      case DIB_METRIC_BINARY_ACCURACY: v = ((zz > threshold ? 1.f : 0.f) == t) ? 1.f : 0.f; break;
      default:                                                  // DIB_METRIC_BINARY_CROSSENTROPY
        if (from_logits) v = fmaxf(zz, 0.f) - zz * t + log1pf(expf(-fabsf(zz)));
        else {
          const float pc = fminf(fmaxf(zz, ep), 1.f - ep);
          v = -(t * logf(pc + ep) + (1.f - t) * logf(1.f - pc + ep));
        }
    }
    s += v;
  }
  return s / (float)out_dim;
}

// fixed-order sum of v over the CTA (shuffle tree per warp, then the warps in order); the result is valid in thread 0
__device__ __forceinline__ float cta_sum(float v, float* red) {
  v = dib_warp_sum(v);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
  __syncthreads();
  float r = 0.f;
  if (threadIdx.x == 0)
    for (int i = 0; i < kWarps; ++i) r += red[i];
  __syncthreads();
  return r;
}

// Grid-stride over the rows, one row per lane.  Mean metrics accumulate (sum w m, sum w) in registers; a confusion metric
// finds the row's bucket by binary search over its float32 threshold table in shared memory and adds w to the warp's own
// histogram: the lanes of a warp that hit the same bucket are summed in lane order by the lowest of them, so every float sum
// has a fixed order.  Each CTA writes its partial tail; the last CTA to finish (an integer counter) sums the partials in CTA
// order into the tail and resets the counter.  No float atomics: the tail depends on n and the data only.
__global__ void __launch_bounds__(kThreads)
dib_metrics_kernel(const DibMetricTable t, const float* __restrict__ z, const float* __restrict__ y, int out_dim, long long n,
                   const float* __restrict__ w, float* __restrict__ part, unsigned int* __restrict__ counter,
                   float* __restrict__ tail) {
  extern __shared__ float sm[];
  float* thr = sm;                                   // [buckets]: metric k's table at boff[k] (T of its T + 1 entries)
  float* hist = thr + t.buckets;                     // [warps][2 * buckets]: metric k's [neg | pos] at 2 * boff[k]
  float* stage = hist + kWarps * 2 * t.buckets;      // [warps][32]
  __shared__ float red[kWarps];
  __shared__ bool last;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  for (int k = 0; k < t.count; ++k)
    if (t.kind[k] == DIB_METRIC_CONFUSION)
      for (int i = threadIdx.x; i < t.nthr[k]; i += kThreads)
        thr[t.boff[k] + i] = t.nthr[k] == 1 ? t.threshold[k] : auc_threshold(i, t.nthr[k]);
  for (int i = threadIdx.x; i < kWarps * 2 * t.buckets; i += kThreads) hist[i] = 0.f;
  __syncthreads();

  float acc[2 * kDibMaxMetrics];
#pragma unroll
  for (int k = 0; k < 2 * kDibMaxMetrics; ++k) acc[k] = 0.f;
  float* my_hist = hist + warp * 2 * t.buckets;
  float* my_stage = stage + warp * 32;
  const long long stride = (long long)gridDim.x * kThreads;
  for (long long base = (long long)blockIdx.x * kThreads + warp * 32; base < n; base += stride) {   // warp-uniform
    const long long row = base + lane;
    const bool valid = row < n;
    const float wr = valid && w ? w[row] : 1.f;
    const float z0 = valid ? z[row * out_dim] : 0.f;
    const float sig = t.sigmoid ? 1.f / (1.f + expf(-z0)) : 0.f;       // sigmoid(z) in fp32, libm expf, once per row
#pragma unroll
    for (int k = 0; k < kDibMaxMetrics; ++k) {
      if (k >= t.count) break;
      const float wk = t.weighted[k] ? wr : 1.f;
      if (t.kind[k] != DIB_METRIC_CONFUSION) {
        if (valid) {
          const float m = mean_metric(t.kind[k], t.from_logits[k], t.threshold[k], z, y, row, out_dim);
          acc[2 * k] += wk * m;
          acc[2 * k + 1] += wk;
        }
        continue;
      }
      const int T = t.nthr[k];
      int b = -1;
      if (valid) {
        const float p = t.from_logits[k] ? sig : z0;
        const float* tk = thr + t.boff[k];
        int lo = 0, hi = T;                 // lo = #{j : p > t_j} (the table ascends; NaN exceeds none)
        while (lo < hi) {
          const int mid = (lo + hi) >> 1;
          if (p > tk[mid]) lo = mid + 1; else hi = mid;
        }
        b = (y[row] != 0.f ? T + 1 : 0) + lo;
      }
      my_stage[lane] = wk;
      __syncwarp();
      const unsigned grp = __match_any_sync(0xffffffffu, b);
      if (b >= 0 && lane == __ffs(grp) - 1) {
        float s = 0.f;
        for (unsigned m = grp; m; m &= m - 1) s += my_stage[__ffs(m) - 1];
        my_hist[2 * t.boff[k] + b] += s;
      }
      __syncwarp();
    }
  }
  __syncthreads();

  float* my_part = part + (long long)blockIdx.x * t.tail;
#pragma unroll
  for (int k = 0; k < kDibMaxMetrics; ++k) {
    if (k >= t.count) break;
    if (t.kind[k] == DIB_METRIC_CONFUSION) continue;
    const float s0 = cta_sum(acc[2 * k], red);
    const float s1 = cta_sum(acc[2 * k + 1], red);
    if (threadIdx.x == 0) { my_part[t.off[k]] = s0; my_part[t.off[k] + 1] = s1; }
  }
  for (int k = 0; k < t.count; ++k) {
    if (t.kind[k] != DIB_METRIC_CONFUSION) continue;
    const int len = 2 * (t.nthr[k] + 1);
    for (int i = threadIdx.x; i < len; i += kThreads) {
      float s = 0.f;
      for (int q = 0; q < kWarps; ++q) s += hist[q * 2 * t.buckets + 2 * t.boff[k] + i];
      my_part[t.off[k] + i] = s;
    }
  }
  __threadfence();
  __syncthreads();
  if (threadIdx.x == 0) last = atomicAdd(counter, 1u) == gridDim.x - 1;
  __syncthreads();
  if (!last) return;
  __threadfence();
  for (int i = threadIdx.x; i < t.tail; i += kThreads) {
    float s = 0.f;
    for (unsigned c = 0; c < gridDim.x; ++c) s += __ldcg(part + (long long)c * t.tail + i);
    tail[i] = s;
  }
  if (threadIdx.x == 0) *counter = 0u;
}

__global__ void dib_metrics_update_tail_kernel(const float* __restrict__ tail, double* __restrict__ acc, int count) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < count) acc[i] += (double)tail[i];
}

}  // namespace

cudaError_t dib_launch_metrics(const DibMetricTable& t, const float* z, const float* y, int out_dim, int64_t n, const float* w,
                               float* part, unsigned int* counter, float* tail, cudaStream_t st) {
  if (t.count <= 0) return cudaSuccess;
  if (n <= 0) return cudaMemsetAsync(tail, 0, sizeof(float) * (size_t)t.tail, st);
  long long grid = DIB_CEIL_DIV((long long)n, (long long)kThreads * kRowsPerThread);
  if (grid > kDibMetricMaxCtas) grid = kDibMetricMaxCtas;
  const size_t smem = sizeof(float) * ((size_t)t.buckets * (1 + 2 * kWarps) + kWarps * 32);
  dib_metrics_kernel<<<(unsigned)grid, kThreads, smem, st>>>(t, z, y, out_dim, (long long)n, w, part, counter, tail);
  dib_note_launch();
  return cudaGetLastError();
}

cudaError_t dib_metrics_prepare(const DibMetricTable& t) {
  const size_t smem = sizeof(float) * ((size_t)t.buckets * (1 + 2 * kWarps) + kWarps * 32);
  if (smem <= 48 * 1024) return cudaSuccess;        // more dynamic shared memory needs the opt-in (current device)
  return cudaFuncSetAttribute(dib_metrics_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
}

cudaError_t dib_launch_metrics_update_tail(const float* tail, double* acc, int count, cudaStream_t st) {
  if (count <= 0) return cudaSuccess;
  dib_metrics_update_tail_kernel<<<DIB_CEIL_DIV(count, 256), 256, 0, st>>>(tail, acc, count);
  dib_note_launch();
  return cudaGetLastError();
}
