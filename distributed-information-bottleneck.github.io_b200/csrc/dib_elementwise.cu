// dib_elementwise.cu -- the non-GEMM kernels of the fp32 parity path: positional encoding, reparameterisation
// + per-feature KL, compiled loss/metric + its gradient, deterministic reductions, Keras-Adam, Bhattacharyya.
#include "dib_common.cuh"
#include "dib_kernels.h"

namespace {

constexpr int kRowsPerBlock = 256;

// block-wide deterministic sum (fixed shuffle tree + fixed-order warp combine); result valid in thread 0.
__device__ __forceinline__ float block_sum_256(float v, float* smem8) {
  v = dib_warp_sum(v);
  const int w = threadIdx.x >> 5, l = threadIdx.x & 31;
  if (l == 0) smem8[w] = v;
  __syncthreads();
  float r = 0.f;
  if (threadIdx.x == 0) {
    const int nw = (blockDim.x + 31) >> 5;
    for (int i = 0; i < nw; ++i) r += smem8[i];
  }
  __syncthreads();
  return r;
}

// ------------------------------------------------------------------------------------------------
// models.py:22-23 PositionalEncoding.call: concat([x] + [sin(f x) for f in (2,4,8,16)], -1), block-major
// per feature, written into the zero-padded operand of the first encoder layer.
// ------------------------------------------------------------------------------------------------
__global__ void dib_pe_kernel(const float* __restrict__ x, int ldx, int x_col_shift, const int* __restrict__ col_src,
                              const int* __restrict__ col_freq, int col_begin, int ncols, float* __restrict__ pe,
                              int ldpe, int pe_col_shift, long long n, int round_out,
                              const int* __restrict__ row_index, const int* __restrict__ col_feat, long long n_src) {
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= n * ncols) return;
  const long long row = idx / ncols;
  const int col = col_begin + (int)(idx % ncols);
  const int src = col_src[col];
  float v = 0.f;
  if (src >= 0) {
    long long srow = row;
    if (row_index) {   // per-feature row gather (visualization.py:17-28 picks different rows for every feature)
      srow = row_index[(long long)col_feat[col] * n + row];
      srow = srow < 0 ? 0 : (srow >= n_src ? n_src - 1 : srow);
    }
    const float xv = x[srow * ldx + (src - x_col_shift)];
    const int f = col_freq[col];
    v = f == 0 ? xv : sinf((float)f * xv);
  }
  pe[row * ldpe + (col - pe_col_shift)] = dib_maybe_round(v, round_out);
}

// ------------------------------------------------------------------------------------------------
// models.py:106-112: split (mu, logvar), u = mu + exp(logvar/2)*eps, KL_i partial sums.
// One thread per (row, feature); blockIdx.y = feature.
// ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(kRowsPerBlock)
dib_reparam_fwd_kernel(DibReparamArgs a, float* __restrict__ emb, int ldemb, float* __restrict__ user_emb,
                       float* __restrict__ kl_part, int nblk_stride) {
  __shared__ float red[8];
  const long long row = (long long)blockIdx.x * kRowsPerBlock + threadIdx.x;
  const int f = blockIdx.y, E = a.E;
  float kl = 0.f;
  const bool pad = a.set_sizes && row < a.n && (int)(row % a.set_len) >= a.set_sizes[row / a.set_len];
  if (pad) {                       // a padding particle of a padded set: u = 0, outside the KL
    for (int e = 0; e < E; ++e) {
      emb[row * ldemb + f * E + e] = 0.f;
      if (user_emb) user_emb[row * ((long long)a.F * E) + f * E + e] = 0.f;
    }
    if (f == a.F - 1)
      for (int c = a.F * E; c < ldemb; ++c) emb[row * ldemb + c] = 0.f;
  } else if (row < a.n) {
    const float* o = a.enc_out + (long long)f * a.feat_stride + row * a.ldo;
    float* dst = emb + row * ldemb + f * E;
    float* udst = user_emb ? user_emb + row * ((long long)a.F * E) + f * E : nullptr;
    const float* ep = a.eps ? a.eps + (row * a.F + f) * E : nullptr;
    for (int e0 = 0; e0 < E; e0 += 4) {
      float nrm[4];
      if (!ep) dib_philox_normal4(a.seed, a.step + (a.step_dev ? a.step_dev[0] : 0u), a.sample_offset + (uint64_t)row, (uint32_t)f, (uint32_t)(e0 >> 2), nrm);
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const int e = e0 + j;
        if (e < E) {
          const float mu = o[e], lv = o[E + e];
          const float s = expf(0.5f * lv);
          const float z = ep ? ep[e] : nrm[j];
          const float u = fmaf(s, z, mu);
          kl += 0.5f * (mu * mu + expf(lv) - lv - 1.f);
          dst[e] = dib_maybe_round(u, a.round_out);
          if (udst) udst[e] = u;
        }
      }
    }
    if (f == a.F - 1)
      for (int c = a.F * E; c < ldemb; ++c) emb[row * ldemb + c] = 0.f;
  }
  const float s = block_sum_256(kl, red);
  if (threadIdx.x == 0) kl_part[(long long)f * nblk_stride + blockIdx.x] = s;
}

// d mu = du + beta*mu/B ; d logvar = du*eps*0.5*sigma + beta*0.5*(exp(logvar)-1)/B
__global__ void __launch_bounds__(kRowsPerBlock)
dib_reparam_bwd_kernel(DibReparamArgs a, const float* __restrict__ d_emb, int ldemb, const float* __restrict__ beta_dev,
                       float inv_batch, float* __restrict__ d_out) {
  const long long row = (long long)blockIdx.x * kRowsPerBlock + threadIdx.x;
  if (row >= a.n) return;
  const int f = blockIdx.y, E = a.E;
  const float bs = beta_dev[0] * inv_batch;
  const float* o = a.enc_out + (long long)f * a.feat_stride + row * a.ldo;
  float* dq = d_out + (long long)f * a.feat_stride + row * a.ldo;
  if (a.set_sizes && (int)(row % a.set_len) >= a.set_sizes[row / a.set_len]) {   // padding particle: no gradient
    for (int c = 0; c < a.ldo; ++c) dq[c] = 0.f;
    return;
  }
  const float* du = d_emb + row * ldemb + f * E;
  const float* ep = a.eps ? a.eps + (row * a.F + f) * E : nullptr;
  for (int e0 = 0; e0 < E; e0 += 4) {
    float nrm[4];
    if (!ep) dib_philox_normal4(a.seed, a.step + (a.step_dev ? a.step_dev[0] : 0u), a.sample_offset + (uint64_t)row, (uint32_t)f, (uint32_t)(e0 >> 2), nrm);
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int e = e0 + j;
      if (e < E) {
        const float mu = o[e], lv = o[E + e], g = du[e];
        const float s = expf(0.5f * lv);
        const float z = ep ? ep[e] : nrm[j];
        dq[e] = dib_maybe_round(fmaf(bs, mu, g), a.round_out);
        dq[E + e] = dib_maybe_round(fmaf(g * z, 0.5f * s, bs * 0.5f * (expf(lv) - 1.f)), a.round_out);
      }
    }
  }
  for (int c = 2 * E; c < a.ldo; ++c) dq[c] = 0.f;
}

// ------------------------------------------------------------------------------------------------
// compiled loss (Keras, data.py:65 / :343 / MSE), metrics=['accuracy'] (data.py:67) and d loss / d z_out.
// One thread per row.
// ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(kRowsPerBlock)
dib_loss_kernel(int loss, int out_act, float alpha, const float* __restrict__ pred, int ldp, const float* __restrict__ y,
                int out_dim, long long n, float inv_batch, float* __restrict__ d_pred, float* __restrict__ user_pred,
                float* __restrict__ loss_part, float* __restrict__ acc_part, int round_out) {
  __shared__ float red[8];
  const long long row = (long long)blockIdx.x * kRowsPerBlock + threadIdx.x;
  float l = 0.f, acc = 0.f;
  if (row < n) {
    const float* z = pred + row * ldp;
    float* dz = d_pred ? d_pred + row * ldp : nullptr;
    if (user_pred)
      for (int j = 0; j < out_dim; ++j) user_pred[row * out_dim + j] = z[j];
    if (y && loss == DIB_LOSS_EXTERNAL) {
      // the caller's d(task loss)/d(prediction); only the output activation's derivative is applied here
      if (dz)
        for (int j = 0; j < out_dim; ++j)
          dz[j] = dib_maybe_round(y[row * out_dim + j] * dib_act_grad(out_act, z[j], alpha), round_out);
    } else if (y) {
      const float inv_out = 1.f / (float)out_dim;
      if (loss == DIB_LOSS_SPARSE_CE_LOGITS) {
        const int label = (int)y[row];
        float m = z[0]; int am = 0;
        for (int j = 1; j < out_dim; ++j) if (z[j] > m) { m = z[j]; am = j; }
        float se = 0.f;
        for (int j = 0; j < out_dim; ++j) se += expf(z[j] - m);
        l = m + logf(se) - z[label];
        acc = (am == label) ? 1.f : 0.f;
        if (dz) {
          const float inv_se = 1.f / se;
          for (int j = 0; j < out_dim; ++j) {
            const float g = expf(z[j] - m) * inv_se - (j == label ? 1.f : 0.f);
            dz[j] = dib_maybe_round(g * inv_batch * dib_act_grad(out_act, z[j], alpha), round_out);
          }
        }
      } else {
        const float* yy = y + row * out_dim;
        for (int j = 0; j < out_dim; ++j) {
          const float zz = z[j];
          const float g = dib_loss_add(loss, zz, yy[j], l, acc);
          if (dz) dz[j] = dib_maybe_round(g * inv_out * inv_batch * dib_act_grad(out_act, zz, alpha), round_out);
        }
        l *= inv_out;
        acc *= inv_out;
      }
    }
    if (dz)
      for (int c = out_dim; c < ldp; ++c) dz[c] = 0.f;
  }
  const float ls = block_sum_256(l, red);
  const float as = block_sum_256(acc, red);
  if (threadIdx.x == 0) { loss_part[blockIdx.x] = ls; acc_part[blockIdx.x] = as; }
}

// stats = [ sum_b KL_i (F) | sum_b task loss | sum_b accuracy | n ]; one block, one WARP per item (fixed lane-strided
// order + fixed shuffle tree -> deterministic), no block-wide barriers.
__global__ void __launch_bounds__(256)
dib_finalize_stats_kernel(const float* __restrict__ kl_part, int nblk_stride, int nblk_kl, const float* __restrict__ loss_part,
                          const float* __restrict__ acc_part, int nblk_loss, int F, long long n, int has_y,
                          float* __restrict__ out) {
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, nwarps = blockDim.x >> 5;
  for (int item = warp; item < F + 2; item += nwarps) {
    const float* src; int cnt;
    if (item < F) { src = kl_part + (long long)item * nblk_stride; cnt = nblk_kl; }
    else { src = item == F ? loss_part : acc_part; cnt = has_y ? nblk_loss : 0; }
    float v = 0.f;
    for (int i = lane; i < cnt; i += 32) v += src[i];
    v = dib_warp_sum(v);
    if (lane == 0) out[item] = v;
  }
  if (threadIdx.x == 0) out[F + 2] = (float)n;
}

__global__ void dib_reduce_partials_kernel(const float* __restrict__ part, long long split_stride, int nsplit,
                                           long long count, float* __restrict__ out) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= count) return;
  float s = 0.f;                       // fixed summation order (deterministic); loads batched 8 deep for latency
  int k = 0;
  for (; k + 8 <= nsplit; k += 8) {
    float v[8];
#pragma unroll
    for (int u = 0; u < 8; ++u) v[u] = part[(long long)(k + u) * split_stride + i];
#pragma unroll
    for (int u = 0; u < 8; ++u) s += v[u];
  }
  for (; k < nsplit; ++k) s += part[(long long)k * split_stride + i];
  out[i] = s;
}

__global__ void dib_round_copy_kernel(const float* __restrict__ src, float* __restrict__ dst, long long count) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < count) dst[i] = dib_round_tf32(src[i]);
}

__global__ void dib_copy2d_kernel(const float* __restrict__ src, int lds, float* __restrict__ dst, int ldd, int cols,
                                  long long n) {
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= n * cols) return;
  const long long r = idx / cols; const int c = (int)(idx % cols);
  dst[r * ldd + c] = src[r * lds + c];
}

// ------------------------------------------------------------------------------------------------
// tf.keras.optimizers.Adam (epsilon outside the bias correction); step counter and lr on the device.
// ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256)
dib_adam_kernel(float* __restrict__ w, const float* __restrict__ g, float* __restrict__ m, float* __restrict__ v,
                long long count, const float* __restrict__ lr_dev, const int32_t* __restrict__ step_dev, float b1,
                float b2, float eps) {
  __shared__ float s_lr_t;
  if (threadIdx.x == 0) {
    const double t = (double)(step_dev[0] + 1);
    s_lr_t = lr_dev[0] * (float)sqrt(1.0 - pow((double)b2, t)) / (float)(1.0 - pow((double)b1, t));
  }
  __syncthreads();
  const float lr_t = s_lr_t, c1 = 1.f - b1, c2 = 1.f - b2;
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= count) return;
  const float gi = g[i];
  float mi = m[i], vi = v[i];
  mi += (gi - mi) * c1;
  vi += (gi * gi - vi) * c2;
  m[i] = mi; v[i] = vi;
  w[i] -= lr_t * mi / (sqrtf(vi) + eps);
}

__global__ void dib_inc_step_kernel(int32_t* step_dev) { step_dev[0] += 1; }

// ------------------------------------------------------------------------------------------------
// utils.py:177-212 (Bhattacharyya, mode 0) and utils.py:213-247 (KL(1||2), mode 1) between two sets of diagonal
// Gaussians in closed form, + exp(-D) (visualization.py:34).  One thread per (i, j); blockIdx.y = group (feature).
// ------------------------------------------------------------------------------------------------
__global__ void dib_pairwise_gauss_kernel(int mode, const float* __restrict__ ml1, long long ld1, long long gstride1,
                                          long long n, const float* __restrict__ ml2, long long ld2, long long gstride2,
                                          long long m, int E, float* __restrict__ out_dist, float* __restrict__ out_comp) {
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= n * m) return;
  const long long g = blockIdx.y;
  const long long i = idx / m, j = idx % m;
  const float* a = ml1 + g * gstride1 + i * ld1;
  const float* b = ml2 + g * gstride2 + j * ld2;
  float D;
  if (mode == 0) {
    float t1 = 0.f, t2 = 0.f;
    for (int e = 0; e < E; ++e) {
      const float d = a[e] - b[e];
      const float la = a[E + e], lb = b[E + e];
      const float sbar = 0.5f * (expf(la) + expf(lb));
      t1 += d * d / sbar;
      t2 += logf(sbar) - 0.5f * (la + lb);
    }
    D = 0.125f * t1 + 0.5f * t2;
  } else {
    float acc = 0.f;
    for (int e = 0; e < E; ++e) {
      const float d = b[e] - a[e];
      const float la = a[E + e], lb = b[E + e];
      acc += (lb - la - 1.f) + expf(la - lb) + d * d * expf(-lb);
    }
    D = 0.5f * acc;
  }
  const long long o = g * n * m + idx;
  if (out_dist) out_dist[o] = D;
  if (out_comp) out_comp[o] = expf(-D);
}

// Keras Mean-metric aggregation over the batches of an epoch (see dib_metrics_update in dib_b200.h).
__global__ void dib_metrics_update_kernel(const float* __restrict__ stats, const float* __restrict__ beta_dev,
                                          float* __restrict__ acc, int F, float kl_exponent, float kl_scale) {
  __shared__ float red[8];
  const float n = stats[F + 2];
  float v = 0.f;
  for (int i = threadIdx.x; i < F; i += blockDim.x) {
    const float s = stats[i];
    if (n > 0.f) acc[i] += s / n;
    v += s;
  }
  const float klsum = block_sum_256(v, red);
  if (threadIdx.x == 0 && n > 0.f) {
    // models.py:118 beta * sum KL (sample-weighted: n * batch mean), or nb-chaos' beta * L * KL^p
    acc[F] += stats[F] + (kl_exponent == 1.f ? beta_dev[0] * kl_scale * klsum
                                            : n * beta_dev[0] * kl_scale * powf(klsum / n, kl_exponent));
    acc[F + 1] += stats[F + 1];
    acc[F + 2] += n;
    acc[F + 3] += 1.f;
  }
}

// ------------------------------------------------------------------------------------------------
// next row f1 -- utils.py:36-65 compute_batch: InfoNCE / leave-one-out bounds of one encoder on one batch.
// One block per sample i: u_i = mu_i + sigma_i eps_i in shared memory, threads stride over j, log-space
// (max, sum) reduction for logsumexp over all j and over j != i.  row_out[i] = (lower_i, upper_i).
// ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256)
dib_mi_rows_kernel(const float* __restrict__ ml, int n, int E, const float* __restrict__ eps, unsigned long long seed,
                   unsigned int step, float* __restrict__ row_out) {
  extern __shared__ float u_s[];            // [E]
  __shared__ float red_m[8], red_s[8], red_s2[8], s_diag;
  const int i = blockIdx.x, tid = threadIdx.x;
  for (int e = tid; e < E; e += blockDim.x) {
    float z;
    if (eps) z = eps[(long long)i * E + e];
    else { float nrm[4]; dib_philox_normal4(seed, step, (unsigned long long)i, 0u, (unsigned)(e >> 2), nrm); z = nrm[e & 3]; }
    u_s[e] = fmaf(expf(0.5f * ml[(long long)i * 2 * E + E + e]), z, ml[(long long)i * 2 * E + e]);
  }
  __syncthreads();
  const float cst = -0.5f * (float)E * 1.8378770664093453f;       // -E/2 log(2 pi)
  // pass 1: log p_ij for this thread's j's, running max
  float lmax = -INFINITY;
  for (int j = tid; j < n; j += blockDim.x) {
    const float* mj = ml + (long long)j * 2 * E;
    float q = 0.f, sl = 0.f;
    for (int e = 0; e < E; ++e) { const float lv = mj[E + e], dlt = u_s[e] - mj[e]; q = fmaf(dlt * dlt, expf(-lv), q); sl += lv; }
    const float lp = -0.5f * q - 0.5f * sl + cst;
    if (j == i) s_diag = lp;
    lmax = fmaxf(lmax, lp);
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) lmax = fmaxf(lmax, __shfl_xor_sync(0xffffffffu, lmax, o));
  if ((tid & 31) == 0) red_m[tid >> 5] = lmax;
  __syncthreads();
  float m = red_m[0];
  for (int w = 1; w < (blockDim.x >> 5); ++w) m = fmaxf(m, red_m[w]);
  // pass 2: sums of exp(lp - m) over all j and over j != i (recomputing lp keeps registers/smem independent of n)
  float s_all = 0.f, s_off = 0.f;
  for (int j = tid; j < n; j += blockDim.x) {
    const float* mj = ml + (long long)j * 2 * E;
    float q = 0.f, sl = 0.f;
    for (int e = 0; e < E; ++e) { const float lv = mj[E + e], dlt = u_s[e] - mj[e]; q = fmaf(dlt * dlt, expf(-lv), q); sl += lv; }
    const float ex = expf(-0.5f * q - 0.5f * sl + cst - m);
    s_all += ex;
    if (j != i) s_off += ex;
  }
  s_all = dib_warp_sum(s_all); s_off = dib_warp_sum(s_off);
  if ((tid & 31) == 0) { red_s[tid >> 5] = s_all; red_s2[tid >> 5] = s_off; }
  __syncthreads();
  if (tid == 0) {
    float a = 0.f, b = 0.f;
    for (int w = 0; w < (blockDim.x >> 5); ++w) { a += red_s[w]; b += red_s2[w]; }
    const float logn = logf((float)n);
    row_out[2 * i] = s_diag - (m + logf(a) - logn);              // InfoNCE term      (utils.py:59-61)
    row_out[2 * i + 1] = s_diag - (m + logf(b) - logn);          // leave-one-out term (utils.py:63-64; still / bs)
  }
}

__global__ void __launch_bounds__(256)
dib_mi_mean_kernel(const float* __restrict__ row_out, int n, float* __restrict__ out2) {
  __shared__ double red[2][8];
  double a = 0.0, b = 0.0;
  for (int i = threadIdx.x; i < n; i += blockDim.x) { a += (double)row_out[2 * i]; b += (double)row_out[2 * i + 1]; }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) { a += __shfl_xor_sync(0xffffffffu, a, o); b += __shfl_xor_sync(0xffffffffu, b, o); }
  if ((threadIdx.x & 31) == 0) { red[0][threadIdx.x >> 5] = a; red[1][threadIdx.x >> 5] = b; }
  __syncthreads();
  if (threadIdx.x == 0) {
    double sa = 0.0, sb2 = 0.0;
    for (int w = 0; w < 8; ++w) { sa += red[0][w]; sb2 += red[1][w]; }
    out2[0] = (float)(sa / n); out2[1] = (float)(sb2 / n);
  }
}

inline unsigned nblocks(long long work, int per) { return (unsigned)((work + per - 1) / per); }

}  // namespace

cudaError_t dib_launch_pe(const float* x, int ldx, int x_col_shift, const int* col_src, const int* col_freq,
                          int col_begin, int col_end, float* pe, int ldpe, int pe_col_shift, int64_t n, int round_out,
                          cudaStream_t st, const int* row_index, const int* col_feat, int64_t n_src) {
  const int ncols = col_end - col_begin;
  if (n <= 0 || ncols <= 0) return cudaSuccess;
  dib_pe_kernel<<<nblocks((long long)n * ncols, 256), 256, 0, st>>>(x, ldx, x_col_shift, col_src, col_freq, col_begin,
                                                                   ncols, pe, ldpe, pe_col_shift, n, round_out,
                                                                   row_index, col_feat, n_src);
  dib_note_launch();
  return cudaGetLastError();
}

cudaError_t dib_launch_reparam_fwd(const DibReparamArgs& a, float* emb, int ldemb, float* user_emb, float* kl_part,
                                   int nblk_stride, cudaStream_t st) {
  if (a.n <= 0) return cudaSuccess;
  dim3 grid(nblocks(a.n, kRowsPerBlock), a.F);
  dib_reparam_fwd_kernel<<<grid, kRowsPerBlock, 0, st>>>(a, emb, ldemb, user_emb, kl_part, nblk_stride);
  dib_note_launch();
  return cudaGetLastError();
}

cudaError_t dib_launch_reparam_bwd(const DibReparamArgs& a, const float* d_emb, int ldemb, const float* beta_dev,
                                   float inv_batch, float* d_out, cudaStream_t st) {
  if (a.n <= 0) return cudaSuccess;
  dim3 grid(nblocks(a.n, kRowsPerBlock), a.F);
  dib_reparam_bwd_kernel<<<grid, kRowsPerBlock, 0, st>>>(a, d_emb, ldemb, beta_dev, inv_batch, d_out);
  dib_note_launch();
  return cudaGetLastError();
}

cudaError_t dib_launch_loss(int loss, int out_act, float alpha, const float* pred, int ldp, const float* y, int out_dim,
                            int64_t n, float inv_batch, float* d_pred, float* user_pred, float* loss_part,
                            float* acc_part, int round_out, cudaStream_t st) {
  if (n <= 0) return cudaSuccess;
  dib_loss_kernel<<<nblocks(n, kRowsPerBlock), kRowsPerBlock, 0, st>>>(loss, out_act, alpha, pred, ldp, y, out_dim, n,
                                                                      inv_batch, d_pred, user_pred, loss_part, acc_part,
                                                                      round_out);
  dib_note_launch();
  return cudaGetLastError();
}

cudaError_t dib_launch_finalize_stats(const float* kl_part, int nblk_stride, int nblk_kl, const float* loss_part,
                                      const float* acc_part, int nblk_loss, int F, int64_t n, int has_y, float* out_stats,
                                      cudaStream_t st) {
  dib_finalize_stats_kernel<<<1, 256, 0, st>>>(kl_part, nblk_stride, nblk_kl, loss_part, acc_part, nblk_loss, F, n,
                                               has_y, out_stats);
  dib_note_launch();
  return cudaGetLastError();
}

cudaError_t dib_launch_reduce_partials(const float* part, long long split_stride, int nsplit, int64_t count, float* out,
                                       cudaStream_t st) {
  if (count <= 0) return cudaSuccess;
  dib_reduce_partials_kernel<<<nblocks(count, 256), 256, 0, st>>>(part, split_stride, nsplit, count, out);
  dib_note_launch();
  return cudaGetLastError();
}

cudaError_t dib_launch_copy2d(const float* src, int lds, float* dst, int ldd, int cols, int64_t n, cudaStream_t st) {
  if (n <= 0 || cols <= 0) return cudaSuccess;
  dib_copy2d_kernel<<<nblocks((long long)n * cols, 256), 256, 0, st>>>(src, lds, dst, ldd, cols, n);
  dib_note_launch();
  return cudaGetLastError();
}

cudaError_t dib_launch_adam(float* params, const float* grads, float* m, float* v, int64_t count, const float* lr_dev,
                            int32_t* step_dev, float b1, float b2, float eps, cudaStream_t st) {
  if (count > 0)
    dib_adam_kernel<<<nblocks(count, 256), 256, 0, st>>>(params, grads, m, v, count, lr_dev, step_dev, b1, b2, eps);
  dib_note_launch();
  dib_inc_step_kernel<<<1, 1, 0, st>>>(step_dev);
  dib_note_launch();
  return cudaGetLastError();
}

cudaError_t dib_launch_pairwise_gauss(int mode, const float* ml1, int64_t ld1, int64_t gstride1, int64_t n,
                                      const float* ml2, int64_t ld2, int64_t gstride2, int64_t m, int E, int groups,
                                      float* out_dist, float* out_comp, cudaStream_t st) {
  if (n <= 0 || m <= 0 || groups <= 0) return cudaSuccess;
  dim3 grid(nblocks((long long)n * m, 128), groups);
  dib_pairwise_gauss_kernel<<<grid, 128, 0, st>>>(mode, ml1, ld1, gstride1, n, ml2, ld2, gstride2, m, E, out_dist, out_comp);
  dib_note_launch();
  return cudaGetLastError();
}

cudaError_t dib_launch_metrics_update(const float* stats, const float* beta_dev, float* acc, int F, float kl_exponent,
                                      float kl_scale, cudaStream_t st) {
  dib_metrics_update_kernel<<<1, 256, 0, st>>>(stats, beta_dev, acc, F, kl_exponent, kl_scale);
  dib_note_launch();
  return cudaGetLastError();
}

cudaError_t dib_launch_round_copy(const float* src, float* dst, int64_t count, cudaStream_t st) {
  if (count <= 0) return cudaSuccess;
  dib_round_copy_kernel<<<nblocks(count, 256), 256, 0, st>>>(src, dst, count);
  dib_note_launch();
  return cudaGetLastError();
}

namespace {
struct ReduceSegsArg { DibReduceSeg seg[kDibMaxReduceSegs]; int first_block[kDibMaxReduceSegs + 1]; int flat[kDibMaxReduceSegs]; int nseg; };
// A list of independent fixed-order reductions in one launch.  Two mappings per segment: FLAT (few rows, many outputs -- the
// batch-split weight-gradient partials): one output per thread, rows summed in order, loads batched 8 deep, coalesced across the
// block; TALL (many rows, few outputs -- per-tile / per-CTA column sums): 32 outputs x 8 row lanes per block.
__global__ void __launch_bounds__(256)
dib_reduce_segments_kernel(const ReduceSegsArg A) {
  __shared__ float red[8][32];
  int sidx = 0;
#pragma unroll
  for (int k = 1; k < kDibMaxReduceSegs; ++k) if (k < A.nseg && (int)blockIdx.x >= A.first_block[k]) sidx = k;
  const DibReduceSeg S = A.seg[sidx];
  const int blk = (int)blockIdx.x - A.first_block[sidx];
  if (A.flat[sidx]) {
    const long long i = (long long)blk * 256 + threadIdx.x;
    if (i >= S.count) return;
    float s = 0.f;
    int k = 0;
    for (; k + 8 <= S.nrows; k += 8) {
      float v[8];
#pragma unroll
      for (int u = 0; u < 8; ++u) v[u] = S.src[(long long)(k + u) * S.row_stride + i];
#pragma unroll
      for (int u = 0; u < 8; ++u) s += v[u];
    }
    for (; k < S.nrows; ++k) s += S.src[(long long)k * S.row_stride + i];
    S.dst[i] = s * S.scale;
    return;
  }
  const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;
  const long long i = (long long)blk * 32 + tx;
  float s = 0.f;
  if (i < S.count) {
    int r = ty;
    for (; r + 56 < S.nrows; r += 64) {
      float v[8];
#pragma unroll
      for (int u = 0; u < 8; ++u) v[u] = S.src[(long long)(r + 8 * u) * S.row_stride + i];
#pragma unroll
      for (int u = 0; u < 8; ++u) s += v[u];
    }
    for (; r < S.nrows; r += 8) s += S.src[(long long)r * S.row_stride + i];
  }
  red[ty][tx] = s;
  __syncthreads();
  if (ty == 0 && i < S.count) {
    float t = 0.f;
    for (int k = 0; k < 8; ++k) t += red[k][tx];
    S.dst[i] = t * S.scale;
  }
}
}  // namespace

cudaError_t dib_launch_reduce_segments(const DibReduceSeg* segs, int nseg, cudaStream_t st) {
  for (int base = 0; base < nseg; base += kDibMaxReduceSegs) {
    ReduceSegsArg A{};
    int nb = 0, n = 0;
    for (int k = base; k < nseg && n < kDibMaxReduceSegs; ++k) {
      if (segs[k].count <= 0) continue;
      A.seg[n] = segs[k]; A.first_block[n] = nb;
      A.flat[n] = (segs[k].nrows <= 64 && segs[k].count >= 4096) ? 1 : 0;
      nb += (int)((segs[k].count + (A.flat[n] ? 255 : 31)) / (A.flat[n] ? 256 : 32));
      ++n;
    }
    A.first_block[n] = nb; A.nseg = n;
    if (n == 0) continue;
    dib_reduce_segments_kernel<<<nb, 256, 0, st>>>(A);
    dib_note_launch();
  }
  return cudaGetLastError();
}

cudaError_t dib_launch_mi_sandwich(const float* mu_logvar, int64_t n, int E, const float* eps, uint64_t seed, uint32_t step,
                                   float* row_scratch, float* out2, cudaStream_t st) {
  if (n <= 0) return cudaSuccess;
  dib_mi_rows_kernel<<<(unsigned)n, 256, E * sizeof(float), st>>>(mu_logvar, (int)n, E, eps, seed, step, row_scratch);
  dib_note_launch();
  dib_mi_mean_kernel<<<1, 256, 0, st>>>(row_scratch, (int)n, out2);
  dib_note_launch();
  return cudaGetLastError();
}


// ================================================================================================
// custom-step variants of the front end (SURVEY 8f3)
// ================================================================================================
namespace {

__global__ void dib_add_logvar_offset_kernel(float* __restrict__ enc_out, long long feat_stride, int ldo, int F, int E,
                                             long long n, float offset, int feature) {
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  const int nf = feature >= 0 ? 1 : F;
  if (idx >= n * E * nf) return;
  const int e = (int)(idx % E);
  const long long row = (idx / E) % n;
  const int f = feature >= 0 ? feature : (int)(idx / ((long long)E * n));
  enc_out[(long long)f * feat_stride + row * ldo + E + e] += offset;
}

// nb-bool cell 4: call(inputs) = concat([inputs * mu_scaling, ones_like(inputs) * logvar], -1)
__global__ void dib_simple_enc_fwd_kernel(const float* __restrict__ x, int ldx, const int* __restrict__ x_off,
                                          const float* __restrict__ params, float* __restrict__ enc_out, long long feat_stride,
                                          int ldo, int F, int E, long long n, int feature, int x_is_feature_only,
                                          const int* __restrict__ row_index, long long n_src) {
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  const int nf = feature >= 0 ? 1 : F;
  if (idx >= n * E * nf) return;
  const int e = (int)(idx % E);
  const long long row = (idx / E) % n;
  const int f = feature >= 0 ? feature : (int)(idx / ((long long)E * n));
  long long srow = row;
  if (row_index) { srow = row_index[(long long)f * n + row]; srow = srow < 0 ? 0 : (srow >= n_src ? n_src - 1 : srow); }
  const float xv = x[srow * ldx + (x_is_feature_only ? 0 : x_off[f]) + e];
  float* o = enc_out + (long long)f * feat_stride + row * ldo;
  o[e] = xv * params[2 * f];
  o[E + e] = params[2 * f + 1];
  if (e == 0) for (int c = 2 * E; c < ldo; ++c) o[c] = 0.f;
}

// grid (F, nsplit): deterministic block sums of d_mu * x and d_logvar over one batch slice
__global__ void __launch_bounds__(256)
dib_simple_enc_wgrad_kernel(const float* __restrict__ x, int ldx, const int* __restrict__ x_off, const float* __restrict__ d_out,
                            long long feat_stride, int ldo, int E, long long n, int rows_per_split, float* __restrict__ part,
                            long long split_stride) {
  __shared__ float red[8];
  const int f = blockIdx.x, split = blockIdx.y;
  const long long r0 = (long long)split * rows_per_split, r1 = min(n, r0 + rows_per_split);
  float gm = 0.f, gl = 0.f;
  for (long long row = r0 + threadIdx.x; row < r1; row += blockDim.x) {
    const float* dq = d_out + (long long)f * feat_stride + row * ldo;
    const float* xr = x + row * ldx + x_off[f];
    for (int e = 0; e < E; ++e) { gm = fmaf(dq[e], xr[e], gm); gl += dq[E + e]; }
  }
  const float sm = block_sum_256(gm, red);
  const float sl = block_sum_256(gl, red);
  if (threadIdx.x == 0) {
    part[(long long)split * split_stride + 2 * f] = sm;
    part[(long long)split * split_stride + 2 * f + 1] = sl;
  }
}

__global__ void dib_beta_eff_kernel(const float* __restrict__ stats, int F, float inv_global_batch, const float* __restrict__ beta_dev,
                                    float exponent, float scale, float* __restrict__ out) {
  if (threadIdx.x != 0 || blockIdx.x != 0) return;
  float kl = 0.f;
  for (int i = 0; i < F; ++i) kl += stats[i];
  kl *= inv_global_batch;
  out[0] = beta_dev[0] * scale * (exponent == 1.f ? 1.f : exponent * powf(kl, exponent - 1.f));
}

}  // namespace

cudaError_t dib_launch_add_logvar_offset(float* enc_out, long long feat_stride, int ldo, int F, int E, int64_t n, float offset,
                                         int feature, cudaStream_t st) {
  const long long total = (long long)n * E * (feature >= 0 ? 1 : F);
  if (total <= 0 || offset == 0.f) return cudaSuccess;
  dib_add_logvar_offset_kernel<<<(unsigned)((total + 255) / 256), 256, 0, st>>>(enc_out, feat_stride, ldo, F, E, n, offset, feature);
  dib_note_launch();
  return cudaGetLastError();
}

cudaError_t dib_launch_simple_enc_fwd(const float* x, int ldx, const int* x_off_dev, const float* params, float* enc_out,
                                      long long feat_stride, int ldo, int F, int E, int64_t n, int feature, int x_is_feature_only,
                                      const int* row_index, int64_t n_src, cudaStream_t st) {
  const long long total = (long long)n * E * (feature >= 0 ? 1 : F);
  if (total <= 0) return cudaSuccess;
  dib_simple_enc_fwd_kernel<<<(unsigned)((total + 255) / 256), 256, 0, st>>>(x, ldx, x_off_dev, params, enc_out, feat_stride, ldo,
                                                                             F, E, n, feature, x_is_feature_only, row_index, n_src);
  dib_note_launch();
  return cudaGetLastError();
}

cudaError_t dib_launch_simple_enc_wgrad(const float* x, int ldx, const int* x_off_dev, const float* d_out, long long feat_stride,
                                        int ldo, int F, int E, int64_t n, int nsplit, int rows_per_split, float* part,
                                        long long split_stride, cudaStream_t st) {
  dib_simple_enc_wgrad_kernel<<<dim3(F, nsplit), 256, 0, st>>>(x, ldx, x_off_dev, d_out, feat_stride, ldo, E, n, rows_per_split,
                                                               part, split_stride);
  dib_note_launch();
  return cudaGetLastError();
}

cudaError_t dib_launch_beta_eff(const float* stats, int F, float inv_global_batch, const float* beta_dev, float exponent,
                                float scale, float* beta_eff_dev, cudaStream_t st) {
  dib_beta_eff_kernel<<<1, 32, 0, st>>>(stats, F, inv_global_batch, beta_dev, exponent, scale, beta_eff_dev);
  dib_note_launch();
  return cudaGetLastError();
}

// ================================================================================================
// next row f1, batched: utils.estimate_mi_sandwich_bounds (utils.py:10-73) for G = features x evaluation batches groups of
// n encoder outputs in ONE launch, accumulated in float64 like the reference (utils.py:40-41 casts to float64).
//   log p(u_i | x_j) = -1/2 sum_e (u_ie - mu_je)^2 exp(-lv_je) - 1/2 sum_e lv_je - E/2 log(2 pi)
//   lower = mean_i [ lp_ii - (logsumexp_j lp_ij - log n) ],  upper = the same without the diagonal term in the sum.
// One thread per row i (u_i in a conflict-free shared-memory column), the (mu_j, exp(-lv_j), c_j) of 16 columns j staged
// per step in shared memory (broadcast reads), one online logsumexp per row.  grid = (ceil(n / 128), G).
// ================================================================================================
namespace {

constexpr int kMiRows = 128, kMiTJ = 16, kMiMaxE = 64;

__global__ void __launch_bounds__(kMiRows)
dib_mi_batched_kernel(const float* __restrict__ ml, int n, int E, const float* __restrict__ eps, unsigned long long seed,
                      int batches_per_feature, double* __restrict__ row_out) {
  extern __shared__ double sm[];                 // [kMiTJ][E] mu | [kMiTJ][E] inverse variance | [kMiTJ] c_j | [E][kMiRows] u
  double* s_mu = sm; double* s_iv = sm + kMiTJ * E; double* s_c = sm + 2 * kMiTJ * E;
  double* u = sm + 2 * kMiTJ * E + kMiTJ + threadIdx.x;          // u[e] lives at u[e * kMiRows]
  const int g = blockIdx.y, tid = threadIdx.x;
  const int i = blockIdx.x * kMiRows + tid;
  const bool live = i < n;
  const float* mlg = ml + (long long)g * n * 2 * E;
  const int f = g / batches_per_feature, b = g % batches_per_feature;
  const unsigned long long gseed = (seed << 8) + (unsigned long long)f;      // the per-feature stream of the looped API
  if (live) {
    const float* mi = mlg + (long long)i * 2 * E;
#pragma unroll 4
    for (int e0 = 0; e0 < E; e0 += 4) {
      float nrm[4];
      if (!eps) dib_philox_normal4(gseed, (unsigned)b, (unsigned long long)i, 0u, (unsigned)(e0 >> 2), nrm);
      for (int k = 0; k < 4 && e0 + k < E; ++k) {
        const int e = e0 + k;
        const double z = eps ? (double)eps[((long long)g * n + i) * E + e] : (double)nrm[k];
        u[e * kMiRows] = (double)mi[e] + exp(0.5 * (double)mi[E + e]) * z;    // utils.py:43-45, in float64
      }
    }
  }
  const double cst = -0.5 * (double)E * 1.8378770664093454836;                // -E/2 log(2 pi)
  double m = -1e300, s_all = 0.0, s_off = 0.0, diag = 0.0;
  for (int j0 = 0; j0 < n; j0 += kMiTJ) {
    __syncthreads();
    for (int t = tid; t < kMiTJ * E; t += kMiRows) {
      const int jj = t / E, e = t - jj * E, j = j0 + jj;
      if (j < n) { s_mu[t] = (double)mlg[(long long)j * 2 * E + e]; s_iv[t] = exp(-(double)mlg[(long long)j * 2 * E + E + e]); }
    }
    if (tid < kMiTJ && j0 + tid < n) {
      double sl = 0.0;
      for (int e = 0; e < E; ++e) sl += (double)mlg[(long long)(j0 + tid) * 2 * E + E + e];
      s_c[tid] = -0.5 * sl + cst;
    }
    __syncthreads();
    if (!live) continue;
    const int jn = min(kMiTJ, n - j0);
    for (int jj = 0; jj < jn; ++jj) {
      double q = 0.0;
#pragma unroll 8
      for (int e = 0; e < E; ++e) { const double d = u[e * kMiRows] - s_mu[jj * E + e]; q = fma(d * d, s_iv[jj * E + e], q); }
      const double lp = -0.5 * q + s_c[jj];
      if (lp > m) { const double r = exp(m - lp); s_all *= r; s_off *= r; m = lp; }
      const double ex = exp(lp - m);
      s_all += ex;
      if (j0 + jj == i) diag = lp; else s_off += ex;
    }
  }
  if (live) {
    const double logn = log((double)n);
    double* o = row_out + ((long long)g * n + i) * 2;
    o[0] = diag - (m + log(s_all) - logn);                                    // InfoNCE term       (utils.py:59-61)
    o[1] = diag - (m + log(s_off) - logn);                                    // leave-one-out term (utils.py:63-64; still / bs)
  }
}

__global__ void __launch_bounds__(256)
dib_mi_batched_mean_kernel(const double* __restrict__ row_out, int n, double* __restrict__ out) {
  __shared__ double red[2][8];
  const int g = blockIdx.x;
  double a = 0.0, b = 0.0;
  for (int i = threadIdx.x; i < n; i += blockDim.x) { a += row_out[((long long)g * n + i) * 2]; b += row_out[((long long)g * n + i) * 2 + 1]; }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) { a += __shfl_xor_sync(0xffffffffu, a, o); b += __shfl_xor_sync(0xffffffffu, b, o); }
  if ((threadIdx.x & 31) == 0) { red[0][threadIdx.x >> 5] = a; red[1][threadIdx.x >> 5] = b; }
  __syncthreads();
  if (threadIdx.x == 0) {
    double sa = 0.0, sb2 = 0.0;
    for (int w = 0; w < 8; ++w) { sa += red[0][w]; sb2 += red[1][w]; }
    out[2 * g] = sa / n; out[2 * g + 1] = sb2 / n;
  }
}

}  // namespace

cudaError_t dib_launch_mi_sandwich_batched(const float* mu_logvar, int groups, int64_t n, int E, const float* eps, uint64_t seed,
                                           int batches_per_feature, double* row_scratch, double* out, cudaStream_t st) {
  if (n <= 0 || groups <= 0) return cudaSuccess;
  if (E > kMiMaxE) return cudaErrorInvalidValue;
  const size_t smem = (size_t)(2 * kMiTJ * E + kMiTJ + kMiRows * E) * sizeof(double);
  static bool attr = false;
  if (!attr) {
    cudaError_t e = cudaFuncSetAttribute(dib_mi_batched_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                         (int)((2 * kMiTJ * kMiMaxE + kMiTJ + kMiRows * kMiMaxE) * sizeof(double)));
    if (e != cudaSuccess) return e;
    attr = true;
  }
  dib_mi_batched_kernel<<<dim3((unsigned)((n + kMiRows - 1) / kMiRows), groups), kMiRows, smem, st>>>(
      mu_logvar, (int)n, E, eps, seed, batches_per_feature < 1 ? 1 : batches_per_feature, row_scratch);
  dib_note_launch();
  dib_mi_batched_mean_kernel<<<groups, 256, 0, st>>>(row_scratch, (int)n, out);
  dib_note_launch();
  return cudaGetLastError();
}


// ================================================================================================
// the other Keras optimizers (train.py:41,128 tf.keras.optimizers.get(name)) and the stand-alone positional encoding
// ================================================================================================
namespace {

__global__ void dib_sgd_kernel(float* __restrict__ w, const float* __restrict__ g, float* __restrict__ v, long long count,
                               const float* __restrict__ lr_dev, float momentum, int nesterov) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= count) return;
  const float lr = lr_dev[0], gi = g[i];
  if (momentum == 0.f) { w[i] -= lr * gi; return; }
  const float vi = momentum * v[i] - lr * gi;
  v[i] = vi;
  w[i] += nesterov ? momentum * vi - lr * gi : vi;
}

__global__ void dib_rmsprop_kernel(float* __restrict__ w, const float* __restrict__ g, float* __restrict__ ms, float* __restrict__ mom,
                                   long long count, const float* __restrict__ lr_dev, float rho, float momentum, float eps) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= count) return;
  const float lr = lr_dev[0], gi = g[i];
  const float m2 = rho * ms[i] + (1.f - rho) * gi * gi;
  ms[i] = m2;
  const float mo = momentum * mom[i] + lr * gi / sqrtf(m2 + eps);
  mom[i] = mo;
  w[i] -= mo;
}

__global__ void dib_pe_plain_kernel(const float* __restrict__ x, long long n, int d, int nfreq, float* __restrict__ out) {
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  const int W = d * nfreq;
  if (idx >= n * W) return;
  const long long row = idx / W;
  const int col = (int)(idx - row * W), blk = col / d, k = col - blk * d;
  const float xv = x[row * d + k];
  out[idx] = blk == 0 ? xv : sinf((float)(1 << blk) * xv);
}

}  // namespace

cudaError_t dib_launch_optimizer(int kind, float* params, const float* grads, float* s1, float* s2, int64_t count,
                                 const float* lr_dev, int32_t* step_dev, float h0, float h1, float h2, cudaStream_t st) {
  if (count > 0) {
    if (kind == 0) dib_sgd_kernel<<<nblocks(count, 256), 256, 0, st>>>(params, grads, s1, count, lr_dev, h0, h1 != 0.f);
    else dib_rmsprop_kernel<<<nblocks(count, 256), 256, 0, st>>>(params, grads, s1, s2, count, lr_dev, h0, h1, h2);
    dib_note_launch();
  }
  dib_inc_step_kernel<<<1, 1, 0, st>>>(step_dev);
  dib_note_launch();
  return cudaGetLastError();
}

cudaError_t dib_launch_pe_plain(const float* x, int64_t n, int d, int nfreq, float* out, cudaStream_t st) {
  const long long total = (long long)n * d * nfreq;
  if (total <= 0) return cudaSuccess;
  dib_pe_plain_kernel<<<nblocks(total, 256), 256, 0, st>>>(x, n, d, nfreq, out);
  dib_note_launch();
  return cudaGetLastError();
}


// ================================================================================================
// Keras Dropout on the hidden activations of the feature encoders (nb-radial cell 5), Philox-keyed
// ================================================================================================
namespace {

__global__ void dib_dropout_kernel(const float* __restrict__ src, float* __restrict__ dst, long long feat_stride, int ld, int width,
                                   int F, long long n, float rate, unsigned long long seed, unsigned int step,
                                   const unsigned int* __restrict__ step_dev, unsigned long long sample_offset, int layer,
                                   int feature, int backward, int round_out) {
  const int nq = (width + 3) >> 2;
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  const int nf = feature >= 0 ? 1 : F;
  if (idx >= n * nq * nf) return;
  const int quad = (int)(idx % nq);
  const long long row = (idx / nq) % n;
  const int f = feature >= 0 ? feature : (int)(idx / ((long long)nq * n));
  const long long base = (long long)f * feat_stride + row * ld + 4 * quad;
  float keep[4] = {1.f, 1.f, 1.f, 1.f};
  if (rate > 0.f) {
    const unsigned long long sample = sample_offset + (unsigned long long)row;
    uint32_t r[4];
    dib_philox4x32_10((uint32_t)sample, (uint32_t)(sample >> 32) ^ ((uint32_t)f << 8),
                      0x80000000u | ((uint32_t)layer << 24) | (uint32_t)quad, step + (step_dev ? step_dev[0] : 0u),
                      (uint32_t)seed, (uint32_t)(seed >> 32), r);
    const float inv_keep = 1.f / (1.f - rate);
#pragma unroll
    for (int k = 0; k < 4; ++k) keep[k] = (((float)(r[k] >> 8) + 0.5f) * 5.9604644775390625e-08f >= rate) ? inv_keep : 0.f;
  }
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    if (4 * quad + k < width) {
      const float v = (backward ? dst[base + k] : src[base + k]) * keep[k];
      dst[base + k] = dib_maybe_round(v, round_out);
    }
  }
}

}  // namespace

cudaError_t dib_launch_dropout(const float* src, float* dst, long long feat_stride, int ld, int width, int F, int64_t n, float rate,
                               uint64_t seed, uint32_t step, const uint32_t* step_dev, uint64_t sample_offset, int layer,
                               int feature, int backward, int round_out, cudaStream_t st) {
  const long long total = (long long)n * ((width + 3) / 4) * (feature >= 0 ? 1 : F);
  if (total <= 0) return cudaSuccess;
  dib_dropout_kernel<<<nblocks(total, 256), 256, 0, st>>>(src, dst, feat_stride, ld, width, F, n, rate, seed, step, step_dev,
                                                         sample_offset, layer, feature, backward, round_out);
  dib_note_launch();
  return cudaGetLastError();
}
