// dib_common.cuh -- shared device helpers of the Distributed-IB engine (H100, sm_90a).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "../../include/dib_b200.h"

#define DIB_CEIL_DIV(a, b) (((a) + (b) - 1) / (b))
#define DIB_ROUND_UP(a, b) (DIB_CEIL_DIV(a, b) * (b))

// ---------------------------------------------------------------------------------------------
// activations (tf.keras.activations.get(name) as used at models.py:76,82); derivatives are taken
// from the OUTPUT h = act(z), which is what the backward kernels have in HBM / shared memory.
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ float dib_act(int act, float z, float alpha) {
  switch (act) {
    case DIB_ACT_RELU: return fmaxf(z, 0.f);
    case DIB_ACT_TANH: return tanhf(z);
    case DIB_ACT_LEAKY_RELU: return z > 0.f ? z : alpha * z;
    case DIB_ACT_SIGMOID: return 1.f / (1.f + expf(-z));
    case DIB_ACT_ELU: return z > 0.f ? z : expm1f(z);
    default: return z;
  }
}

// the same for the 16-bit-operand kernels, whose outputs are rounded to 11 / 8 significant bits anyway: tanh / sigmoid / elu on
// the SFU approximations (tanh.approx: relative error ~2^-11; ex2 / rcp.approx ~2^-22) instead of the libm routines
__device__ __forceinline__ float dib_act16(int act, float z, float alpha) {
  switch (act) {
    case DIB_ACT_RELU: return fmaxf(z, 0.f);
    case DIB_ACT_TANH: { float t; asm("tanh.approx.f32 %0, %1;" : "=f"(t) : "f"(z)); return t; }
    case DIB_ACT_LEAKY_RELU: return z > 0.f ? z : alpha * z;
    case DIB_ACT_SIGMOID: return __fdividef(1.f, 1.f + __expf(-z));
    case DIB_ACT_ELU: return z > 0.f ? z : __expf(z) - 1.f;
    default: return z;
  }
}

__device__ __forceinline__ float dib_act_grad(int act, float h, float alpha) {
  switch (act) {
    case DIB_ACT_RELU: return h > 0.f ? 1.f : 0.f;
    case DIB_ACT_TANH: return 1.f - h * h;
    case DIB_ACT_LEAKY_RELU: return h > 0.f ? 1.f : alpha;
    case DIB_ACT_SIGMOID: return h * (1.f - h);
    case DIB_ACT_ELU: return h > 0.f ? 1.f : h + 1.f;
    default: return 1.f;
  }
}

// One output of the compiled loss and metrics=['accuracy'] for target t: BCE on logits, keras.backend.binary_crossentropy
// on probabilities, or MSE (every other loss).  Adds the loss term to l and the accuracy hit to acc and returns d loss / d z,
// all unscaled: the callers apply 1/out, 1/batch and the output activation's derivative.  The sum is formed inside each
// branch so that it contracts with the term (l += d * d is one FMA).  A caller that wants the bare term starts from l = -0.f,
// which x + -0.f leaves exact.  The softmax cross-entropy couples the outputs and stays with its callers.
__device__ __forceinline__ float dib_loss_add(int loss, float z, float t, float& l, float& acc) {
  float g;
  if (loss == DIB_LOSS_BCE_LOGITS) { l += fmaxf(z, 0.f) - z * t + log1pf(expf(-fabsf(z))); g = 1.f / (1.f + expf(-z)) - t; }
  else if (loss == DIB_LOSS_BCE_PROBS) {
    const float ep = 1e-7f, pc = fminf(fmaxf(z, ep), 1.f - ep);
    l -= t * logf(pc + ep) + (1.f - t) * logf(1.f - pc + ep);
    g = (z > ep && z < 1.f - ep) ? -t / (pc + ep) + (1.f - t) / (1.f - pc + ep) : 0.f;
  } else { const float d = z - t; l += d * d; g = 2.f * d; }
  acc += ((z > 0.5f ? 1.f : 0.f) == t) ? 1.f : 0.f;
  return g;
}

// The same with the loss term weighted by the row's sample weight w (Keras SUM_OVER_BATCH_SIZE: sum_i w_i l_i / n); the
// accuracy hit and d loss / d z stay unweighted (the callers weight d loss / d z through their 1/batch factor).  w enters
// as the last factor of a product term (MSE: d * (d * w)), so that with w = 1 every sum contracts as in dib_loss_add and
// all-ones weights give the unweighted bits.
__device__ __forceinline__ float dib_loss_add_w(int loss, float z, float t, float w, float& l, float& acc) {
  float g;
  if (loss == DIB_LOSS_BCE_LOGITS) { l += (fmaxf(z, 0.f) - z * t + log1pf(expf(-fabsf(z)))) * w; g = 1.f / (1.f + expf(-z)) - t; }
  else if (loss == DIB_LOSS_BCE_PROBS) {
    const float ep = 1e-7f, pc = fminf(fmaxf(z, ep), 1.f - ep);
    l -= (t * logf(pc + ep) + (1.f - t) * logf(1.f - pc + ep)) * w;
    g = (z > ep && z < 1.f - ep) ? -t / (pc + ep) + (1.f - t) / (1.f - pc + ep) : 0.f;
  } else { const float d = z - t; l += d * (d * w); g = 2.f * d; }
  acc += ((z > 0.5f ? 1.f : 0.f) == t) ? 1.f : 0.f;
  return g;
}

// The class a sparse label t names among C, as Keras on a GPU reads it: t is cast to an integer by truncation and is valid
// when -1 < t < C; any other t (NaN included) gives -1, and the callers then return a NaN loss, a NaN d loss / d z for the
// whole row and no accuracy hit.  An accuracy hit is (float)argmax == t, so a label of 2.7 names class 2 but never hits.
__device__ __forceinline__ int dib_sparse_label(float t, int C) { return (t > -1.f && t < (float)C) ? (int)t : -1; }

// 2 KL(N(mu, e^lv) || N(0, 1)) = mu^2 + (e^lv - 1 - lv).  e^lv - 1 - lv = lv^2/2 + lv^3/6 + ... is formed from terms near 1
// and loses all relative accuracy as lv -> 0, which is where high beta drives the unused features; expm1f keeps it above
// |lv| = 1/16 and a short series takes over below (its first dropped term is lv^4/360 relative, under 2^-24), in the way
// dib_neg_log treats -ln(u) near 1.
__device__ __forceinline__ float dib_kl_term(float mu, float lv) {
  const float series = lv * lv * (0.5f + lv * (0.16666667f + lv * (0.041666668f + lv * 0.008333334f)));
  return fmaf(mu, mu, fabsf(lv) < 0.0625f ? series : expm1f(lv) - lv);
}

// dib_loss_add, weighted (W) or not: the one switch the loss epilogues of the WEIGHTED kernel instantiations go through
template <bool W>
__device__ __forceinline__ float dib_loss_add_t(int loss, float z, float t, float w, float& l, float& acc) {
  if constexpr (W) return dib_loss_add_w(loss, z, t, w, l, acc);
  else return dib_loss_add(loss, z, t, l, acc);
}

// ---------------------------------------------------------------------------------------------
// Philox4x32-10 noise; contract documented in oracle/philox.py (the CPU restatement used by tests).
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ void dib_philox4x32_10(uint32_t c0, uint32_t c1, uint32_t c2, uint32_t c3,
                                                  uint32_t k0, uint32_t k1, uint32_t out[4]) {
  const uint32_t M0 = 0xD2511F53u, M1 = 0xCD9E8D57u;
#pragma unroll
  for (int r = 0; r < 10; ++r) {
    const uint32_t hi0 = __umulhi(M0, c0), lo0 = M0 * c0;
    const uint32_t hi1 = __umulhi(M1, c2), lo1 = M1 * c2;
    const uint32_t n0 = hi1 ^ c1 ^ k0, n2 = hi0 ^ c3 ^ k1;
    c0 = n0; c1 = lo1; c2 = n2; c3 = lo0;
    k0 += 0x9E3779B9u; k1 += 0xBB67AE85u;
  }
  out[0] = c0; out[1] = c1; out[2] = c2; out[3] = c3;
}

// -ln(u) for u in (0,1): SFU lg2 away from 1, a short series in (1-u) near 1 (where lg2.approx loses all relative
// accuracy and could even change sign); 1-u is exact because u sits on the 2^-24 grid.
__device__ __forceinline__ float dib_neg_log(float u) {
  const float t = 1.f - u;
  const float series = t * (1.f + t * (0.5f + t * (0.33333334f + t * (0.25f + t * 0.2f))));
  return t < 0.0625f ? series : -__logf(u);
}

// 4 standard normals for (global sample, feature, dims 4*quad .. 4*quad+3) at optimizer step `step`.
__device__ __forceinline__ void dib_philox_normal4(uint64_t seed, uint32_t step, uint64_t sample,
                                                   uint32_t feature, uint32_t quad, float n[4]) {
  uint32_t r[4];
  dib_philox4x32_10((uint32_t)sample, (uint32_t)(sample >> 32) ^ (feature << 8), quad, step,
                    (uint32_t)seed, (uint32_t)(seed >> 32), r);
  const float s = 5.9604644775390625e-08f;  // 2^-24
  const float u0 = ((float)(r[0] >> 8) + 0.5f) * s, u1 = ((float)(r[1] >> 8) + 0.5f) * s;
  const float u2 = ((float)(r[2] >> 8) + 0.5f) * s, u3 = ((float)(r[3] >> 8) + 0.5f) * s;
  // Box-Muller with the SFU approximations (lg2/sqrt/sin/cos.approx): |error| of a sample is a few 1e-7 .. 1e-6,
  // far below what the noise itself means and below every parity tolerance; ~4x fewer instructions than libm.
  const float ra = sqrtf(2.f * dib_neg_log(u0)), rb = sqrtf(2.f * dib_neg_log(u2));
  float sa, ca, sb, cb;
  __sincosf(6.283185307179586f * u1, &sa, &ca);
  __sincosf(6.283185307179586f * u3, &sb, &cb);
  n[0] = ra * ca; n[1] = ra * sa; n[2] = rb * cb; n[3] = rb * sb;
}

// round-to-nearest to the TF32 grid (10 explicit mantissa bits).  kind::tf32 MMAs ignore the low 13 bits of their
// fp32 containers, i.e. TRUNCATE; producers round instead so that the operand error is unbiased (|rel| <= 2^-11).
__device__ __forceinline__ float dib_round_tf32(float x) {
  uint32_t u;
  asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(u) : "f"(x));
  return __uint_as_float(u);
}
__device__ __forceinline__ float dib_maybe_round(float x, int on) { return on ? dib_round_tf32(x) : x; }

// 32 consecutive bytes per thread as two 16-byte accesses (sm_90 has no 32-byte global load / store).  `p` must be 16-byte aligned.
__device__ __forceinline__ void dib_st_global_v8(void* p, uint32_t a, uint32_t b, uint32_t c, uint32_t d, uint32_t e, uint32_t f, uint32_t g, uint32_t h) {
  uint4* q = static_cast<uint4*>(p);
  q[0] = make_uint4(a, b, c, d);
  q[1] = make_uint4(e, f, g, h);
}
__device__ __forceinline__ void dib_st_global_v8(void* p, const uint32_t (&w)[8]) {
  dib_st_global_v8(p, w[0], w[1], w[2], w[3], w[4], w[5], w[6], w[7]);
}
__device__ __forceinline__ void dib_ld_global_v8(const void* p, uint32_t (&w)[8]) {
  const uint4* q = static_cast<const uint4*>(p);
  const uint4 a = q[0], b = q[1];
  w[0] = a.x; w[1] = a.y; w[2] = a.z; w[3] = a.w; w[4] = b.x; w[5] = b.y; w[6] = b.z; w[7] = b.w;
}

__device__ __forceinline__ float dib_warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// the real rows l_s of padded set s.  The sizes live in the caller's device memory and cannot be checked without a sync, so
// every kernel that reads one treats a size outside [1, Lmax] as the nearest bound: forward and backward then agree.
__device__ __forceinline__ int dib_set_len(const int* sizes, long long s, int Lmax) {
  const int l = sizes[s];
  return l < 1 ? 1 : (l > Lmax ? Lmax : l);
}

// ---------------------------------------------------------------------------------------------
// grouped GEMM problem descriptor (one per feature encoder / one for an integration layer).
// Canonical form  Out[R x C] = sum_t Aop[R x T] * Bop[T x C]; see dib_gemm_simt.cu for the three modes.
// All offsets are in floats relative to the base pointers given to the launch.
// ---------------------------------------------------------------------------------------------
struct DibGemmProblem {
  long long a_off, b_off, c_off, x_off;  // x: bias (FWD) / activation source (DGRAD) / bias-grad (WGRAD)
  int lda, ldb, ldc, ldx;
  int T;  // reduction length (FWD: fan-in, DGRAD: fan-out; WGRAD: unused = batch slice)
  int C;  // output columns     (FWD: fan-out, DGRAD: fan-in, WGRAD: fan-out)
  int R;  // output rows for WGRAD (fan-in); unused (batch) otherwise
  int act;  // activation applied (FWD) / differentiated (DGRAD)
};

enum DibGemmMode { DIB_GEMM_FWD = 0, DIB_GEMM_DGRAD = 1, DIB_GEMM_WGRAD = 2 };
