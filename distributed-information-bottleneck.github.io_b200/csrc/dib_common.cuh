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
