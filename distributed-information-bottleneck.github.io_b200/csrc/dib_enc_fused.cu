// dib_enc_fused.cu -- the fused per-feature encoder kernels of the tensor-core mode (sm_90a).
//
// One persistent CTA works on ONE feature at a time: the feature's encoder weights (positional-encoding layer incl. its
// bias row, 128x128 hidden layer, 128x64 (mu|logvar) layer) are TMA-staged into shared memory once and reused for every
// 128-sample tile of that feature.  Per tile the whole chain of models.py:101-112
//     x column -> positional encoding -> Dense(128,act) -> Dense(128,act) -> Dense(2E) -> split (mu, logvar)
//     -> u = mu + exp(logvar/2) eps -> KL partial sums -> emb[:, f*E:(f+1)*E]
// runs on chip: the three contractions are wgmma instructions (16-bit operands with an 11-bit significand = TF32's, fp32
// accumulation in registers), the activations stay in registers (forward: the next MMA's register A operand) or travel
// registers -> shared memory (backward: swizzled operand tiles) and never touch HBM.  Only x (4 B/sample/feature) is read
// and emb is written.
//
// Two MMA warpgroups per CTA; warpgroup g owns rows [64 g, 64 g + 64) of a tile (wgmma M = 64).  Every contraction whose
// reduction runs over the hidden features (forward, dgrad) reads only the warpgroup's own rows, so the two warpgroups
// proceed independently; the weight-gradient contractions of the backward reduce over all 128 samples of the tile and
// meet at barriers of the two.  The backward has a third, producer warpgroup that stages each tile's inputs and noise.
//
// Operand layouts (16-bit): every activation/weight tile is [rows][64-element panels of 128 B] with the 16-byte chunk
// index XORed with (row % 8) -- the SWIZZLE_128B pattern, which for 16-bit types is simultaneously a valid K-major operand
// (rows = M/N, panel = K) and a valid MN-major operand (rows = K, panel = M/N).  That dual view is what lets the backward
// kernel use one copy of h1/h2/dz/W for dgrad (reduction over features) and wgrad (reduction over samples).
#include <cuda.h>
#include <cuda_bf16.h>
#include <cuda_fp16.h>

#include "dib_common.cuh"
#include "dib_kernels.h"
#include "dib_sm90.cuh"

namespace {

using namespace sm90;

constexpr int TM = 128;            // samples per tile
constexpr int HID = 128;           // hidden width of both encoder layers
constexpr int EO = 64;             // 2 * embedding dim
constexpr int K0 = 16;             // padded fan-in of the first layer: [pe (d*nfreq) | 1 (bias) | 0...]
constexpr int kThreads = 256;      // two warpgroups
constexpr int kPanel = TM * 128;   // bytes of one 64-column panel of a 128-row tile (16 KB)

// packed 16-bit weights in global memory, per feature (elements): W0p[16][128] | W1[128][128] | W2[128][64]
// followed by the bias carriers Bb1[16][128] | Bb2[16][64] whose only non-zero row (index w_in, the position of the
// ones column in the first-layer operand) holds b1 / b2: one extra K=16 MMA step adds the bias for free.
constexpr int kW0Elems = K0 * HID, kW1Elems = HID * HID, kW2Elems = HID * EO, kB1Elems = K0 * HID, kB2Elems = K0 * EO;
constexpr int kPackElems = kW0Elems + kW1Elems + kW2Elems + kB1Elems + kB2Elems;

// shared memory map (bytes; swizzled operand tiles 1024-aligned)
constexpr int kOffW1 = 0;
constexpr int kOffW2 = kOffW1 + 2 * kPanel;        // 32 KB
constexpr int kOffW0 = kOffW2 + kPanel;            // 16 KB
constexpr int kOffBb1 = kOffW0 + 2 * K0 * 128;     // 4 KB : W0p = 2 panels x 16 rows x 128 B
constexpr int kOffBb2 = kOffBb1 + 2 * K0 * 128;    // 4 KB : Bb1 likewise
constexpr int kA0Bytes = 2 * TM * 16;              // A0 = [2 k-halves][128 rows][16 B] (no swizzle)
constexpr int kOffA0 = kOffBb2 + K0 * 128;         // 2 KB : Bb2 = 1 panel x 16 rows x 128 B
constexpr int kOffX = kOffA0 + 2 * kA0Bytes;       // 8 KB : two A0 buffers (the backward alternates them; the forward uses one)
constexpr int kOffFwdEnd = kOffX + kThreads * 16;  // 4 KB : x ring, one 16-byte slot per thread (see prefetch_x)
// backward-only tiles (the forward keeps h1 / h2 in registers)
constexpr int kOffH1 = kOffFwdEnd;
constexpr int kOffH2 = kOffH1 + 2 * kPanel;        // h2, later dz1
constexpr int kOffDO = kOffH2 + 2 * kPanel;        // [128 x 64] d(mu | logvar), one panel
constexpr int kOffDZ2 = kOffDO + kPanel;           // [128 x 128]
constexpr int kOffG = kOffDZ2 + 2 * kPanel;        // [128 rows][32] 16-bit d_emb16 of the next tile (TMA, no swizzle)
constexpr int kNzBytes = TM * 32 * 4;              // one tile's noise: [128 rows][32 dims] fp32 (see nz_chunk)
constexpr int kOffNz = kOffG + TM * 64;            // two noise buffers, alternating with the [pe|1] buffers
constexpr int kOffBwdEnd = kOffNz + 2 * kNzBytes;
constexpr int kBwdThreads = kThreads + 128;        // + a producer warpgroup (inputs and noise of the next tile)
static_assert(kOffH1 % 1024 == 0 && kOffDZ2 % 1024 == 0, "operand tiles must be 1024-byte aligned");
static_assert(kOffBwdEnd + 128 + 1024 <= 232448, "backward shared memory exceeds the 227 KB per-block opt-in");

struct EncFusedParams {
  const float* x; int ldx;                 // [n, D]
  const int* x_off;                        // [F] first x column of each feature
  const int* fdim;                         // [F] d_i
  int nfreq;                               // 1 + number of sinusoid blocks (1 = no positional encoding)
  const float* params;                     // fp32 master parameters
  const long long* b1_off; const long long* b2_off;   // [F] offsets of b1, b2 in params
  const float* eps;                        // [n, F, E] or null -> Philox
  unsigned long long seed; unsigned int step; unsigned long long sample_offset;
  const unsigned int* step_dev;            // optional device addend of `step` (CUDA-Graph replay)
  float* emb; int ldemb; float* user_emb;  // outputs (forward); emb may be null when emb16 is given
  uint16_t* emb16; int ldemb16;            // 16-bit (fp16 / bf16) copy of emb for the 16-bit integration path (or null)
  float* kl_part; int kl_stride;           // [F][kl_stride] per-(feature, slot) KL partial sums
  int F; long long n; int act; float alpha;
  int round_emb;
};

// two fp32 -> one 32-bit word of two 16-bit values (a in the low half), saturating instead of producing inf
template <bool BF16>
__device__ __forceinline__ uint32_t pack2(float a, float b) {
  uint32_t r;
  if constexpr (BF16) asm("cvt.rn.satfinite.bf16x2.f32 %0, %1, %2;" : "=r"(r) : "f"(b), "f"(a));
  else asm("cvt.rn.satfinite.f16x2.f32 %0, %1, %2;" : "=r"(r) : "f"(b), "f"(a));
  return r;
}

// same with relu fused into the conversion: max(x, 0) costs no instruction of its own
template <bool BF16>
__device__ __forceinline__ uint32_t pack2_relu(float a, float b) {
  uint32_t r;
  if constexpr (BF16) asm("cvt.rn.relu.satfinite.bf16x2.f32 %0, %1, %2;" : "=r"(r) : "f"(b), "f"(a));
  else asm("cvt.rn.relu.satfinite.f16x2.f32 %0, %1, %2;" : "=r"(r) : "f"(b), "f"(a));
  return r;
}

template <bool BF16>
__device__ __forceinline__ void unpack2(uint32_t u, float& a, float& b) {
  if constexpr (BF16) { const float2 f = __bfloat1622float2(*reinterpret_cast<__nv_bfloat162*>(&u)); a = f.x; b = f.y; }
  else { const float2 f = __half22float2(*reinterpret_cast<__half2*>(&u)); a = f.x; b = f.y; }
}

__device__ __forceinline__ void st_shared_v4(uint32_t addr, uint32_t a, uint32_t b, uint32_t c, uint32_t d) {
  asm volatile("st.shared.v4.b32 [%0], {%1, %2, %3, %4};" ::"r"(addr), "r"(a), "r"(b), "r"(c), "r"(d) : "memory");
}
__device__ __forceinline__ void st_shared_b32(uint32_t addr, uint32_t v) {
  asm volatile("st.shared.b32 [%0], %1;" ::"r"(addr), "r"(v) : "memory");
}
__device__ __forceinline__ uint32_t ld_shared_b32(uint32_t addr) {
  uint32_t v;
  asm volatile("ld.shared.b32 %0, [%1];" : "=r"(v) : "r"(addr) : "memory");
  return v;
}
__device__ __forceinline__ float2 ld_shared_v2f(uint32_t addr) {
  float2 v;
  asm volatile("ld.shared.v2.f32 {%0, %1}, [%2];" : "=f"(v.x), "=f"(v.y) : "r"(addr) : "memory");
  return v;
}

// Position of this thread's accumulator elements in the tile: rows rb and rb + 8, columns 8 j + 2 q (+1).
struct Frag {
  int rb, q;
};
__device__ __forceinline__ Frag frag_of(int tid) {
  const int wg = tid >> 7, wq = (tid >> 5) & 3, lane = tid & 31;
  return Frag{64 * wg + 16 * wq + (lane >> 2), lane & 3};
}

// v, as a value the compiler cannot precompute.  The backward kernel runs at the 255-register limit; addresses and operand
// descriptors derived from such a value are formed where they are used instead of being kept in registers across the tile.
__device__ __forceinline__ uint32_t opaque(uint32_t v) {
  asm volatile("" : "+r"(v));
  return v;
}

// Shared-memory places of a thread's accumulator words in a [128 x 64k] swizzled tile (16-byte chunk index XORed with
// row % 8): word 2 j + h (columns 8 j + 2 q (+1), row rb + 8 h) is at tile + rb * 128 + 4 q + (j / 8) * kPanel + h * 1024
// + ((j % 8) * 16 ^ (rb % 8) * 16).  Bits 4..6 of tile + rb * 128 + 4 q are zero (1024-aligned tile), so the swizzle folds
// into one per-tile word fw.bsw = (tile + rb * 128 + 4 q) ^ (rb % 8) * 16, and the j-th place is one LOP3 with an immediate
// from it: no swizzle term is shared between tiles, where the compiler would keep it in a register through the tile.
struct FragWords {
  uint32_t bsw;
};
__device__ __forceinline__ FragWords frag_words(uint32_t tile, Frag fr) {
  return FragWords{opaque((tile + fr.rb * 128 + 4 * fr.q) ^ ((fr.rb & 7) << 4))};
}
__device__ __forceinline__ uint32_t frag_word_addr(FragWords fw, int j, int h) {
  return (fw.bsw ^ ((j & 7) << 4)) + (j >> 3) * kPanel + h * 1024;
}

// accumulator of a 64 x N tile -> activation -> 16-bit, kept in registers as the next MMA's A operand (the bias is already
// in the accumulator): the accumulator fragment of 8-column block j is the A fragment half i = j % 2 of k step j / 2, so
// a[4 kk .. 4 kk + 3] is the A operand of k step kk (see wgmma_m64n128k16_rs)
template <bool BF16, bool RELU, int N>
__device__ __forceinline__ void frag_to_a(const float (&d)[N / 2], uint32_t (&a)[N / 4], int act, float alpha) {
#pragma unroll
  for (int j = 0; j < N / 8; ++j) {
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const float v0 = d[4 * j + 2 * h], v1 = d[4 * j + 2 * h + 1];
      a[2 * j + h] = RELU ? pack2_relu<BF16>(v0, v1) : pack2<BF16>(dib_act16(act, v0, alpha), dib_act16(act, v1, alpha));
    }
  }
}

// the packed words of such a fragment -> this thread's places in the swizzled shared tile of the warpgroup's 64 x N rows
// (the backward's weight-gradient operands and act').  Each quad of lanes writes one 16-byte chunk of a row: conflict-free
// under the swizzle.
template <int N>
__device__ __forceinline__ void a_to_tile(const uint32_t (&a)[N / 4], uint32_t tile, Frag fr) {
  const FragWords fw = frag_words(tile, fr);
#pragma unroll
  for (int j = 0; j < N / 8; ++j) {
#pragma unroll
    for (int h = 0; h < 2; ++h) st_shared_b32(frag_word_addr(fw, j, h), a[2 * j + h]);
  }
}

// packed 16-bit pair p * (h > 0): relu' applied to two gradients at once (exact: multiplication by 1.0 / 0.0)
template <bool BF16>
__device__ __forceinline__ uint32_t relu_gate2(uint32_t p, uint32_t h) {
  if constexpr (BF16) {
    const __nv_bfloat162 z = __float2bfloat162_rn(0.f);
    __nv_bfloat162 g = __hmul2(*reinterpret_cast<__nv_bfloat162*>(&p), __hgt2(*reinterpret_cast<__nv_bfloat162*>(&h), z));
    return *reinterpret_cast<uint32_t*>(&g);
  } else {
    const __half2 z = __float2half2_rn(0.f);
    __half2 g = __hmul2(*reinterpret_cast<__half2*>(&p), __hgt2(*reinterpret_cast<__half2*>(&h), z));
    return *reinterpret_cast<uint32_t*>(&g);
  }
}

// gradient accumulator (64 x 128) * act'(h) -> 16-bit, packed as the next dgrad MMA's A fragment (layout of frag_to_a); h
// is read back from this thread's own words of the shared tile `htile` that the recomputed forward wrote (relu: as a packed
// comparison, other activations through act'(h)).  a_to_tile stores the result for the weight gradients.
template <bool BF16, bool RELU>
__device__ __forceinline__ void frag_dgrad_to_a(const float (&d)[64], uint32_t htile, uint32_t (&a)[32], Frag fr, int act,
                                                float alpha) {
  const FragWords fw = frag_words(htile, fr);
#pragma unroll
  for (int j = 0; j < 16; ++j) {
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const uint32_t hv = ld_shared_b32(frag_word_addr(fw, j, h));
      const float g0 = d[4 * j + 2 * h], g1 = d[4 * j + 2 * h + 1];
      if constexpr (RELU) {
        a[2 * j + h] = relu_gate2<BF16>(pack2<BF16>(g0, g1), hv);
      } else {
        float h0, h1;
        unpack2<BF16>(hv, h0, h1);
        a[2 * j + h] = pack2<BF16>(g0 * dib_act_grad(act, h0, alpha), g1 * dib_act_grad(act, h1, alpha));
      }
    }
  }
}

// first-layer operand row: [x_0..x_{d-1}, sin(2x).., sin(4x).., ..., 1, 0...] (models.py:22-23 + the ones column
// that carries every layer's bias through the bias-carrier matrices).  xv = the row's feature values.
// sin for the positional encoding: reduce to one period in units of turns, then the SFU (sin.approx of an argument in
// [-pi, pi] is good to ~1e-6 absolute; the reduction adds |arg| * 6e-8) -- no local-memory slow path like sinf's, and far
// below the 16-bit operand rounding (5e-4 relative) that follows.
__device__ __forceinline__ float dib_sin_pe(float a) {
  float t = a * 0.15915494309189535f;
  t -= rintf(t);
  return __sinf(6.283185307179586f * t);
}
constexpr int kMaxFeatDim = 3;     // d * nfreq + 1 <= 16 and nfreq >= 1
template <bool BF16>
__device__ __forceinline__ void write_a0_row(uint32_t a0, int r, int khalf, bool valid, const float (&xv)[kMaxFeatDim], int d,
                                             int nfreq) {
  float f[8];
  const int w_in = d * nfreq;
  int blk = (khalf * 8) / d, j = khalf * 8 - blk * d;      // one division per call; (blk, j) then advance with the column
#pragma unroll
  for (int k = 0; k < 8; ++k) {
    const int col = khalf * 8 + k;
    float v = 0.f;
    if (col < w_in) {
      float xj = xv[0];
#pragma unroll
      for (int q = 1; q < kMaxFeatDim; ++q) if (j == q) xj = xv[q];
      v = blk == 0 ? xj : dib_sin_pe((float)(1 << blk) * xj);
    } else if (col == w_in) {
      v = valid ? 1.f : 0.f;          // rows past the batch end contribute nothing
    }
    f[k] = v;
    if (++j == d) { j = 0; ++blk; }
  }
  st_shared_v4(a0 + khalf * (TM * 16) + r * 16, pack2<BF16>(f[0], f[1]), pack2<BF16>(f[2], f[3]), pack2<BF16>(f[4], f[5]),
               pack2<BF16>(f[6], f[7]));
}

// the [pe|1] operand of one tile: thread t of the CTA stages (row 64 g + t % 64, k-half (t / 64) % 2) of its own warpgroup g
__device__ __forceinline__ int a0_row(int tid) { return 64 * (tid >> 7) + (tid & 63); }

// The x values a thread stages for the tile at row0 are copied into its own 16-byte slot `xs` of the x ring by cp.async
// one tile ahead, so no global-load latency sits in front of stage_a0.  Rows past the batch end copy nothing.  (A TMA
// box cannot do this: the row pitch ldx * 4 B need not be a multiple of 16.)
__device__ __forceinline__ void prefetch_x(const EncFusedParams& P, uint32_t xs, int tid, long long row0, int d, int xo) {
  const long long grow = row0 + a0_row(tid);
  if (grow < P.n) {
    const float* src = P.x + grow * P.ldx + xo;
#pragma unroll
    for (int j = 0; j < kMaxFeatDim; ++j)
      if (j < d) cp_async_4(xs + 4 * j, src + j);
  }
  cp_async_commit();
}
// Waits for this thread's prefetch_x of the tile (slot xslot) and writes its part of [pe|1].  The slot may be refilled
// (prefetch_x of the next tile) as soon as this returns: its values have been consumed by the shared-memory stores.
template <bool BF16>
__device__ __forceinline__ void stage_a0(const EncFusedParams& P, uint32_t a0, const float* xslot, int tid, long long row0,
                                         int d) {
  const int ar = a0_row(tid), khalf = (tid >> 6) & 1;
  const long long grow = row0 + ar;
  cp_async_wait_all();
  float xv[kMaxFeatDim];
#pragma unroll
  for (int j = 0; j < kMaxFeatDim; ++j) xv[j] = (grow < P.n && j < d) ? xslot[j] : 0.f;
  write_a0_row<BF16>(a0, ar, khalf, grow < P.n, xv, d, P.nfreq);
}

// eps for embedding dims (e, e + 1) of row `grow` (e even), explicit tensor or Philox (same keying as dib_elementwise.cu:
// counter word = dim / 4).  The four lanes of a quad hold dims 8 j + 2 q (+1) of two rows, i.e. two Philox quads per row:
// lane q generates quad (2 j + q / 2) of row (q & 1 ? upper : lower) and the quad exchanges the values by shuffles.
__device__ __forceinline__ void noise_pair(const EncFusedParams& P, unsigned int step, long long grow_lo, int f, int j, int q,
                                           int lane, float (&nz)[2][2]) {
  if (P.eps) {
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const long long grow = grow_lo + 8 * h;
      if (grow < P.n) {
        const float2 e = *reinterpret_cast<const float2*>(P.eps + (grow * P.F + f) * 32 + 8 * j + 2 * q);
        nz[h][0] = e.x; nz[h][1] = e.y;
      } else {
        nz[h][0] = nz[h][1] = 0.f;
      }
    }
    return;
  }
  float n4[4];
  dib_philox_normal4(P.seed, step, P.sample_offset + (unsigned long long)(grow_lo + 8 * (q & 1)), (uint32_t)f,
                     (uint32_t)(2 * j + (q >> 1)), n4);
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    const int src = (lane & ~3) | ((q >> 1) << 1) | h;
    float t[4];
#pragma unroll
    for (int k = 0; k < 4; ++k) t[k] = __shfl_sync(0xffffffffu, n4[k], src);
    nz[h][0] = (q & 1) ? t[2] : t[0];
    nz[h][1] = (q & 1) ? t[3] : t[1];
  }
}

struct WeightMaps { CUtensorMap w0, w1, w2, b1, b2; };

// one thread: stage a feature's packed weights (W0p, W1, W2, bias carriers) into shared memory
__device__ __forceinline__ void load_weights(uint32_t sb, const WeightMaps& m, uint32_t bar, int f) {
  mbar_expect_tx(bar, 2 * K0 * 128 + 2 * kPanel + kPanel + 2 * K0 * 128 + K0 * 128);
  tma_load_3d(sb + kOffW0, &m.w0, bar, 0, 0, f);
  tma_load_3d(sb + kOffW0 + K0 * 128, &m.w0, bar, 64, 0, f);
  tma_load_3d(sb + kOffW1, &m.w1, bar, 0, 0, f);
  tma_load_3d(sb + kOffW1 + kPanel, &m.w1, bar, 64, 0, f);
  tma_load_3d(sb + kOffW2, &m.w2, bar, 0, 0, f);
  tma_load_3d(sb + kOffBb1, &m.b1, bar, 0, 0, f);
  tma_load_3d(sb + kOffBb1 + K0 * 128, &m.b1, bar, 64, 0, f);
  tma_load_3d(sb + kOffBb2, &m.b2, bar, 0, 0, f);
}

// ---- operand descriptors.  wg = the issuing warpgroup; its A rows start 64 rows into a tile.
// [pe|1] as A (K-major, no swizzle): 8-row core matrices 128 B apart, k-halves TM*16 B apart
__device__ __forceinline__ uint64_t desc_a0_as_a(uint32_t a0, int wg) { return gmma_desc(a0 + wg * 64 * 16, TM * 16, 128, kLayoutNone); }
// [pe|1] as B over 16 samples from sample 16 kk (MN-major, no swizzle): 8 columns per k-half plane, 8 samples per 128 B
__device__ __forceinline__ uint64_t desc_a0_as_b(uint32_t a0, int kk) { return gmma_desc(a0 + kk * 256, 128, TM * 16, kLayoutNone); }
// activation tile as A (K-major): k step kk of 16 features of the warpgroup's rows
__device__ __forceinline__ uint64_t desc_act_as_a(uint32_t tile, int wg, int kk) {
  return gmma_desc(tile + (kk >> 2) * kPanel + wg * 64 * 128 + (kk & 3) * 32, 16, 1024);
}
// activation tile transposed as A (MN-major): features [64 p, 64 p + 64) of samples [16 kk, 16 kk + 16)
__device__ __forceinline__ uint64_t desc_act_t_as_a(uint32_t tile, int p, int kk) { return gmma_desc(tile + p * kPanel + kk * 2048, kPanel, 1024); }
// activation tile as B over samples (MN-major): all columns, samples [16 kk, 16 kk + 16)
__device__ __forceinline__ uint64_t desc_act_as_b(uint32_t tile, int kk) { return gmma_desc(tile + kk * 2048, kPanel, 1024); }

// the three forward contractions of one warpgroup's 64 rows, each preceded by its bias-carrier step
template <bool BF16>
__device__ __forceinline__ void mma_layer0(float (&d)[64], uint32_t sb, uint32_t a0, int wg) {
  wgmma_m64n128k16<BF16, 0, 1>(d, desc_a0_as_a(a0, wg), gmma_desc(sb + kOffW0, K0 * 128, 1024), 0u);
}
// layers 1 and 2 take h1 / h2 as register A operands (frag_to_a); only their bias-carrier step reads [pe|1] from shared memory
template <bool BF16>
__device__ __forceinline__ void mma_layer1_rs(float (&d)[64], uint32_t sb, const uint32_t (&h1)[32], uint32_t a0, int wg) {
  wgmma_m64n128k16<BF16, 0, 1>(d, desc_a0_as_a(a0, wg), gmma_desc(sb + kOffBb1, K0 * 128, 1024), 0u);
#pragma unroll
  for (int kk = 0; kk < HID / 16; ++kk) {
    const uint32_t a[4] = {h1[4 * kk], h1[4 * kk + 1], h1[4 * kk + 2], h1[4 * kk + 3]};
    wgmma_m64n128k16_rs<BF16, 1>(d, a, gmma_desc(sb + kOffW1 + kk * 2048, kPanel, 1024), 1u);
  }
}
// The backward's recomputed layer 1 reads h1 from its shared tile (after wg_publish): a register A fragment would keep 32
// registers live through the issue, next to the accumulator and the 120 weight-gradient registers, and the backward's MMA
// warpgroups have 240 registers (the producer warpgroup has the rest).
template <bool BF16>
__device__ __forceinline__ void mma_layer1_ss(float (&d)[64], uint32_t sb, uint32_t h1, uint32_t a0, int wg) {
  wgmma_m64n128k16<BF16, 0, 1>(d, desc_a0_as_a(a0, wg), gmma_desc(sb + kOffBb1, K0 * 128, 1024), 0u);
#pragma unroll
  for (int kk = 0; kk < HID / 16; ++kk)
    wgmma_m64n128k16<BF16, 0, 1>(d, desc_act_as_a(h1, wg, kk), gmma_desc(sb + kOffW1 + kk * 2048, kPanel, 1024), 1u);
}
template <bool BF16>
__device__ __forceinline__ void mma_layer2_rs(float (&d)[32], uint32_t sb, const uint32_t (&h2)[32], uint32_t a0, int wg) {
  wgmma_m64n64k16<BF16, 0, 1>(d, desc_a0_as_a(a0, wg), gmma_desc(sb + kOffBb2, K0 * 128, 1024), 0u);
#pragma unroll
  for (int kk = 0; kk < HID / 16; ++kk) {
    const uint32_t a[4] = {h2[4 * kk], h2[4 * kk + 1], h2[4 * kk + 2], h2[4 * kk + 3]};
    wgmma_m64n64k16_rs<BF16, 1>(d, a, gmma_desc(sb + kOffW2 + kk * 2048, kPanel, 1024), 1u);
  }
}

// shared tile written by this warpgroup -> visible to its MMAs
__device__ __forceinline__ void wg_publish(int wg) {
  fence_proxy_async_smem();
  named_bar_sync(1 + wg, 128);
}
// Split-phase hand-off between the backward's two warpgroups: xwg_arrive(e, wg) signals this warpgroup's side of event e
// and does not wait; xwg_wait(e, wg) blocks until the other warpgroup has signalled e.  Named barrier e + g carries
// warpgroup g's signal (128 arriving + 128 waiting threads).  Every event is signalled and waited once per tile, and a
// warpgroup cannot signal an event again before the other has waited for it (each tile ends in a two-sided wait).  The
// fence makes this warpgroup's shared-memory stores visible to the other warpgroup's MMAs.
constexpr uint32_t kEvL0 = 3, kEvDO = 5, kEvDZ2 = 7, kEvDW2 = 9, kEvDZ1 = 11;   // 1, 2: wg_publish
__device__ __forceinline__ void xwg_arrive(uint32_t e, int wg) {
  fence_proxy_async_smem();
  named_bar_arrive(e + wg, 256);
}
__device__ __forceinline__ void xwg_wait(uint32_t e, int wg) { named_bar_sync(e + (wg ^ 1), 256); }

// feature / tile assignment of a persistent CTA: with at least as many CTAs as features, CTA c serves feature c % F and
// its tiles slot, slot + nslots, ...; otherwise it walks features c, c + G, ... with all of their tiles
struct Sched { int f_first, f_step, slot, nslots; };
__device__ __forceinline__ Sched sched_of(int c, int G, int F) {
  if (G >= F) { const int f0 = c % F; return Sched{f0, F * G, c / F, (G - f0 + F - 1) / F}; }
  return Sched{c, G, 0, 1};
}

// ====================================================================================================
// forward: x -> emb, KL partial sums.  71 KB of shared memory, at most 128 registers -> two CTAs per SM, so one CTA's
// epilogue overlaps the other's MMAs.  h1 and h2 never leave registers: each is the register A operand of the next layer.
// ====================================================================================================
template <bool BF16, bool RELU>
__global__ void __launch_bounds__(kThreads, 2)
dib_enc_fused_fwd_kernel(const __grid_constant__ WeightMaps maps, const EncFusedParams P) {
  extern __shared__ uint8_t smem_raw[];
  const uint32_t sb = (smem_u32(smem_raw) + 1023u) & ~1023u;
  uint8_t* sg = smem_raw + (sb - smem_u32(smem_raw));
  float* red_s = reinterpret_cast<float*>(sg + kOffFwdEnd + 64);          // [8 warps]
  const uint32_t bar_w = sb + kOffFwdEnd;

  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, wg = tid >> 7;
  const Frag fr = frag_of(tid);
  const int F = P.F;
  const int ntiles = (int)((P.n + TM - 1) / TM);
  const unsigned int nstep = P.step + (P.step_dev ? P.step_dev[0] : 0u);
  const uint32_t a0 = sb + kOffA0, xs = sb + kOffX + tid * 16;
  const float* xslot = reinterpret_cast<const float*>(sg + kOffX + tid * 16);

  if (tid == 0) {
    tma_prefetch_desc(&maps.w0); tma_prefetch_desc(&maps.w1); tma_prefetch_desc(&maps.w2);
    tma_prefetch_desc(&maps.b1); tma_prefetch_desc(&maps.b2);
    mbar_init(bar_w, 1);
    fence_barrier_init();
  }
  __syncthreads();

  const Sched s = sched_of(blockIdx.x, gridDim.x, F);
  uint32_t fit = 0;
  for (int f = s.f_first; f < F; f += s.f_step, ++fit) {
    if (tid == 0) load_weights(sb, maps, bar_w, f);
    const int d = P.fdim[f], xo = P.x_off[f];
    prefetch_x(P, xs, tid, (long long)s.slot * TM, d, xo);
    float kl_acc = 0.f;
    mbar_wait(bar_w, fit & 1);
    for (int t = s.slot; t < ntiles; t += s.nslots) {
      const long long row0 = (long long)t * TM;
      stage_a0<BF16>(P, a0, xslot, tid, row0, d);
      prefetch_x(P, xs, tid, row0 + (long long)s.nslots * TM, d, xo);
      wg_publish(wg);       // a0 rows of this warpgroup are read only by its own MMAs, which retired in the previous tile
      float acc[64];
      uint32_t ha[32];
      wgmma_fence();
      mma_layer0<BF16>(acc, sb, a0, wg);
      wgmma_commit();
      wgmma_wait<0>();
      wgmma_fence_regs(acc);
      frag_to_a<BF16, RELU, 128>(acc, ha, P.act, P.alpha);
      wgmma_fence();
      mma_layer1_rs<BF16>(acc, sb, ha, a0, wg);
      wgmma_commit();
      wgmma_wait<0>();
      wgmma_fence_regs(acc);
      frag_to_a<BF16, RELU, 128>(acc, ha, P.act, P.alpha);               // h2 over h1
      float acc2[32];
      wgmma_fence();
      mma_layer2_rs<BF16>(acc2, sb, ha, a0, wg);
      wgmma_commit();
      // the noise of this thread's 2 rows x 8 embedding dims while layer 2 runs
      const long long grow_lo = row0 + fr.rb;
      float nz[4][2][2];
#pragma unroll
      for (int j = 0; j < 4; ++j) noise_pair(P, nstep, grow_lo, f, j, fr.q, lane, nz[j]);
      wgmma_wait<0>();
      wgmma_fence_regs(acc2);
      // ---- (mu, logvar) -> reparameterise, KL, emb: columns 8 j + 2 q (+1) are mu, 32 + the same are logvar
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const long long grow = grow_lo + 8 * h;
        if (grow >= P.n) continue;
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          const int e = 8 * j + 2 * fr.q;
          float u[2];
#pragma unroll
          for (int k = 0; k < 2; ++k) {
            const float mu = acc2[4 * j + 2 * h + k], lv = acc2[4 * (j + 4) + 2 * h + k];
            const float sv = __expf(0.5f * lv);      // ex2.approx: relative error 2^-21, far inside the 16-bit operand rounding
            u[k] = fmaf(sv, nz[j][h][k], mu);
            kl_acc += 0.5f * (mu * mu + sv * sv - lv - 1.f);
          }
          if (P.user_emb) *reinterpret_cast<float2*>(P.user_emb + grow * ((long long)F * 32) + f * 32 + e) = make_float2(u[0], u[1]);
          if (P.emb16) *reinterpret_cast<uint32_t*>(P.emb16 + grow * P.ldemb16 + f * 32 + e) = pack2<BF16>(u[0], u[1]);
          if (P.emb) {
            const float2 o = P.round_emb ? make_float2(dib_round_tf32(u[0]), dib_round_tf32(u[1])) : make_float2(u[0], u[1]);
            *reinterpret_cast<float2*>(P.emb + grow * P.ldemb + f * 32 + e) = o;
          }
        }
      }
    }
    // ---- per-(feature, slot) KL partial: fixed-order reduction over the 256 threads
    kl_acc = dib_warp_sum(kl_acc);
    if (lane == 0) red_s[warp] = kl_acc;
    __syncthreads();              // also: both warpgroups are done with this feature's weights
    if (tid == 0) {
      float sum = 0.f;
      for (int i = 0; i < kThreads / 32; ++i) sum += red_s[i];
      P.kl_part[(long long)f * P.kl_stride + s.slot] = sum;
    }
    __syncthreads();
  }
}

// ====================================================================================================
// backward: recompute the forward chain on chip, then dgrad + wgrad of all three layers.
//   d(mu)     = S*du + (beta*S/B)*mu                       (du = d loss / d u from the integration network)
//   d(logvar) = S*du*eps*0.5*sigma + (beta*S/B)*0.5*(sigma^2-1)
//   dz2 = (d(mu|logvar) W2^T) * act'(h2);  dz1 = (dz2 W1^T) * act'(h1)
//   dW2 += h2^T d(mu|logvar);  dW1 += h1^T dz2;  [dW0;db0]^T += dz1^T [pe|1];  db1 = colsum dz2, db2 = colsum d(mu|logvar)
//   (bias gradients = the ones column of [pe|1] used as the B operand: column sums for free)
// S is a power-of-two loss scale that keeps the 16-bit gradient operands in range (fp16); the fp32 accumulators are
// multiplied by 1/S when they are flushed.  The weight-gradient accumulators live in registers for the whole feature:
// warpgroup g owns rows [64 g, 64 g + 64) of dW1, dW2 (and of dW0^T, db1); warpgroup 0 stores db2.  222 KB of shared
// memory: one CTA per SM.
//
// The chain of a warpgroup's rows waits for nothing but its own MMAs (and its own warpgroup):
//   * every MMA that reduces over features (recomputed L1, L2; dgrad G2, G1) reads only the warpgroup's rows.  L1, L2 and
//     G2 take them as register A fragments (h1, h2, dO packed once); the same words are stored to the shared tiles, where
//     only the weight-gradient MMAs (and act') read them.  G1 reads dz2 from its tile (registers are short there);
//   * only the weight-gradient MMAs read the other warpgroup's rows, so they are the only MMAs behind a wait for the other
//     warpgroup.  That wait is split-phase (xwg_arrive / xwg_wait): a warpgroup signals once its rows are stored, issues its
//     dgrad MMAs, and only then waits;
//   * in each backward layer the dgrad MMAs and the weight-gradient MMAs are separate commit groups; the dz epilogue waits
//     only for the dgrad, so the weight-gradient MMAs run under it;
//   * dW0 of tile t retires under the start of tile t + 1 ([pe|1] is double-buffered);
//   * nothing on the chain stages inputs: a third, producer warpgroup writes [pe|1] and the noise of tile t + 1 and issues
//     its d_emb16 TMA (one 8 KB buffer) while the two MMA warpgroups run tile t (see the hand-offs below).
//
// Producer -> consumer hand-offs are mbarriers (the named barriers are taken by the consumers' events).  Each tile k of the
// CTA's sequence (all features' tiles in sched_of order, which both sides walk) uses slot k % 2: a [pe|1] buffer and a noise
// buffer.  Full barriers: a0_full / nz_full[slot] (128 producer threads), bar_g (d_emb16 TMA bytes), bar_w (weights).
// Empty barriers, one arrival per consumer warp (8):
//   * slot_empty[slot]: both warpgroups' dW0 of the tile retired (at the next tile's layer-0 wait, or after the feature's
//     last tile); the noise was read before that, in the tile's dO epilogue;
//   * g_empty: both warpgroups' dO epilogues read d_emb16;
//   * w_empty: both warpgroups' last MMAs of the feature retired: the next feature's weights may be loaded.
// A wait for use u of a buffer is for phase parity u & 1 (full) or (u & 1) ^ 1 (empty: the first use passes at once).
// ====================================================================================================
struct EncFusedBwdParams {
  EncFusedParams f;
  const float* d_emb; int ldd;              // [n, ldd] gradient w.r.t. emb (already scaled by 1/B_global)
  const uint16_t* d_emb16;                  // or: 16-bit gradient already multiplied by the loss scale S (read through gmap)
  const float* beta_dev; float inv_batch; float gscale;
  float* part; long long split_stride;      // weight-gradient partials [slot][P]
  const long long* w0_off; const long long* b0_off; const long long* w1_off; const long long* w2_off;
};

// The backward's feature loop forms the schedule where it is used: both warpgroup roles are at their register limits across
// the tile loop, so what sched_of derives from the CTA index is recomputed per feature instead of kept.  feature_iter = how
// many features this CTA has run before f.
__device__ __forceinline__ Sched sched_here(int F) {
  uint32_t c, G;
  asm volatile("mov.u32 %0, %%ctaid.x;" : "=r"(c));
  asm volatile("mov.u32 %0, %%nctaid.x;" : "=r"(G));
  return sched_of((int)c, (int)G, F);
}
__device__ __forceinline__ uint32_t feature_iter(int f, const Sched& s) { return (uint32_t)((f - s.f_first) / s.f_step); }

// one thread: the [128 rows x 32] block of d_emb16 (feature f, rows from row0) -> shared memory; rows past n read as 0
__device__ __forceinline__ void load_demb16(uint32_t dst, const CUtensorMap* gmap, uint32_t bar, int f, long long row0) {
  mbar_expect_tx(bar, TM * 64);
  tma_load_2d(dst, gmap, bar, f * 32, (int)row0);
}

// Noise buffer of a tile: the 16-byte chunk c (dims 4 c .. 4 c + 3, one Philox quad) of row r sits at r * 128 + (c ^ r % 8) * 16.
// The producer's float4 stores (a warp: 4 rows x 8 chunks) and the consumers' float2 reads of a fragment's pairs (a warp:
// 8 rows x 2 chunks) are both conflict-free; a plain [128][32] layout would make the reads 8-way conflicted.
__device__ __forceinline__ uint32_t nz_chunk(uint32_t nzb, int r, int c) { return nzb + r * 128 + ((c ^ (r & 7)) << 4); }

// the producer's share of tile row0's noise: thread p (of 128) writes the chunks p, p + 128, ... of the [128 x 8] chunks.
// Rows past the batch end are written as zeros (the dO epilogue does not use them).
__device__ __forceinline__ void produce_noise(const EncFusedParams& P, unsigned int nstep, uint32_t nzb, int p, long long row0,
                                              int f) {
#pragma unroll 1
  for (int i = p; i < TM * 8; i += 128) {
    const int r = i >> 3, c = i & 7;
    const long long grow = row0 + r;
    float n4[4] = {0.f, 0.f, 0.f, 0.f};
    if (grow < P.n) {
      if (P.eps) {
        const float* e = P.eps + (grow * P.F + f) * 32 + 4 * c;
        const float2 lo = *reinterpret_cast<const float2*>(e), hi = *reinterpret_cast<const float2*>(e + 2);
        n4[0] = lo.x; n4[1] = lo.y; n4[2] = hi.x; n4[3] = hi.y;
      } else {
        dib_philox_normal4(P.seed, nstep, P.sample_offset + (unsigned long long)grow, (uint32_t)f, (uint32_t)c, n4);
      }
    }
    st_shared_v4(nz_chunk(nzb, r, c), __float_as_uint(n4[0]), __float_as_uint(n4[1]), __float_as_uint(n4[2]),
                 __float_as_uint(n4[3]));
  }
}

// a consumer warp's arrival on an empty barrier, once all its lanes are past their reads
__device__ __forceinline__ void warp_arrive(uint32_t bar) {
  __syncwarp();
  if ((threadIdx.x & 31) == 0) mbar_arrive(bar);
}

template <bool BF16, bool RELU>
__global__ void __launch_bounds__(kBwdThreads, 1)
dib_enc_fused_bwd_kernel(const __grid_constant__ WeightMaps maps, const __grid_constant__ CUtensorMap gmap,
                         const EncFusedBwdParams Q) {
  const EncFusedParams& P = Q.f;
  extern __shared__ uint8_t smem_raw[];
  const uint32_t sb = (smem_u32(smem_raw) + 1023u) & ~1023u;
  const uint32_t bar_w = sb + kOffBwdEnd, w_empty = bar_w + 8, bar_g = bar_w + 16, g_empty = bar_w + 24;
  auto a0_full = [&](uint32_t b) { return bar_w + 32 + 8 * b; };
  auto nz_full = [&](uint32_t b) { return bar_w + 48 + 8 * b; };
  auto slot_empty = [&](uint32_t b) { return bar_w + 64 + 8 * b; };
  // a slot's tile, written by the producer with its [pe|1]: rows inside the batch (<= 128), and whether the weight-gradient
  // MMAs accumulate (all but the feature's first tile; the first one starts them with scale-d = 0)
  auto rows_of = [&](uint32_t b) { return bar_w + 80 + 4 * b; };
  auto wacc_of = [&](uint32_t b) { return bar_w + 88 + 4 * b; };

  const int tid = threadIdx.x, wg = tid >> 7;
  const int F = P.F;
  const uint32_t h1 = sb + kOffH1, h2 = sb + kOffH2, dO = sb + kOffDO, dz2 = sb + kOffDZ2, gbuf = sb + kOffG;
  const float S = Q.gscale;

  if (tid == 0) {
    tma_prefetch_desc(&maps.w0); tma_prefetch_desc(&maps.w1); tma_prefetch_desc(&maps.w2);
    tma_prefetch_desc(&maps.b1); tma_prefetch_desc(&maps.b2);
    if (Q.d_emb16) tma_prefetch_desc(&gmap);
    mbar_init(bar_w, 1);
    mbar_init(w_empty, 8);
    mbar_init(bar_g, 1);
    mbar_init(g_empty, 8);
    for (uint32_t b = 0; b < 2; ++b) { mbar_init(a0_full(b), 128); mbar_init(nz_full(b), 128); mbar_init(slot_empty(b), 8); }
    fence_barrier_init();
  }
  __syncthreads();

  if (wg == 2) {
    // ================= producer: weights, [pe|1], noise and d_emb16 of each tile, one tile ahead of the consumers
    asm volatile("setmaxnreg.dec.sync.aligned.u32 24;");
    // (24 registers: what depends only on the feature or the step is loaded again per tile rather than kept)
    const int p = tid - kThreads;
    uint32_t tk = 0;
    for (int f = sched_here(F).f_first; f < F; f += sched_here(F).f_step) {
      const Sched s = sched_here(F);
      // (the producer's waits are made by all of its threads and only the TMA issue by one: its control flow stays
      // warp-uniform, so that the loop state can live in uniform registers)
      mbar_wait(w_empty, (feature_iter(f, s) & 1) ^ 1);
      if (p == 0) load_weights(sb, maps, bar_w, f);
      for (int t = s.slot; (long long)t * TM < P.n; t += s.nslots, ++tk) {
        const long long row0 = (long long)t * TM;
        const uint32_t b = tk & 1;
        mbar_wait(slot_empty(b), ((tk >> 1) & 1) ^ 1);
        {   // [pe|1]: thread p writes both k-halves of row p
          const int dt = P.fdim[f], xo = P.x_off[f];
          const long long grow = row0 + p;
          float xv[kMaxFeatDim];
#pragma unroll
          for (int j = 0; j < kMaxFeatDim; ++j) xv[j] = (grow < P.n && j < dt) ? P.x[grow * P.ldx + xo + j] : 0.f;
          const uint32_t a0 = sb + kOffA0 + b * kA0Bytes;
          if (p == 0) {
            st_shared_b32(rows_of(b), (uint32_t)min((long long)TM, P.n - row0));
            st_shared_b32(wacc_of(b), t != s.slot);
          }
#pragma unroll 1
          for (int kh = 0; kh < 2; ++kh) write_a0_row<BF16>(a0, p, kh, grow < P.n, xv, dt, P.nfreq);
          fence_proxy_async_smem();        // the consumers' MMAs read it
          mbar_arrive(a0_full(b));
        }
        produce_noise(P, P.step + (P.step_dev ? P.step_dev[0] : 0u), sb + kOffNz + b * kNzBytes, p, row0, f);
        mbar_arrive(nz_full(b));
        if (Q.d_emb16) {
          mbar_wait(g_empty, (tk & 1) ^ 1);
          if (p == 0) load_demb16(gbuf, &gmap, bar_g, f, row0);
        }
      }
    }
    return;
  }
  // ================= consumers: warpgroups 0 and 1
  asm volatile("setmaxnreg.inc.sync.aligned.u32 240;");   // 128 x 24 + 256 x 240 = 384 x 168, what the CTA holds at launch
  const Frag fr = frag_of(tid);
  uint32_t tk = 0;   // tiles run so far; tile tk uses slot tk % 2 and the d_emb16 phase tk % 2
  for (int f = sched_here(F).f_first; f < F; f += sched_here(F).f_step) {
    const Sched s = sched_here(F);
    // The weight-gradient accumulators are started by the first tile's MMAs (scale-d = 0), not by register writes: no
    // instruction but a wgmma may define them while dW0 is in flight across tiles.  A CTA without a tile of the feature
    // flushes zeros.
    float accW1[64], accW2[32], accW0[8], accB1[8], accB2[8];
    mbar_wait(bar_w, feature_iter(f, s) & 1);
    // (the tile count, the schedule and the loss-scaled beta are formed where they are used, and the tile's row count and
    // accumulate flag read from its slot: the consumers' registers are full across the feature loop)
    for (int t = s.slot; (long long)t * TM < P.n; t += sched_here(F).nslots, ++tk) {
      const long long row0 = (long long)t * TM;
      const uint32_t b = tk & 1, bpar = (tk >> 1) & 1;
      const uint32_t a0 = sb + kOffA0 + b * kA0Bytes;
      // ---- recompute the forward of this warpgroup's rows
      mbar_wait(a0_full(b), bpar);
      float acc[64];
      wgmma_fence();
      mma_layer0<BF16>(acc, sb, a0, wg);
      wgmma_commit();
      wgmma_wait<0>();                     // also retires this warpgroup's dW0 of the previous tile
      wgmma_fence_regs(acc); wgmma_fence_regs(accW0);
      xwg_arrive(kEvL0, wg);               // this warpgroup's dW0 of the previous tile (it read all of h2) is done
      if (ld_shared_b32(wacc_of(b))) warp_arrive(slot_empty(b ^ 1));   // ... and with it every read of the previous tile's slot
      uint32_t ha[32];
      frag_to_a<BF16, RELU, 128>(acc, ha, P.act, P.alpha);
      // h1 for dW1 and act'(h1).  The previous tile's dW1 of both warpgroups retired before its kEvDZ1 hand-off.
      a_to_tile<128>(ha, h1, fr);
      // (each MMA chain that starts with scale-d = 0 gets a fresh accumulator: then the values that the previous epilogue
      // consumed are not kept live up to the next MMA's issue)
      float acc1[64];
      wg_publish(wg);
      wgmma_fence();
      mma_layer1_ss<BF16>(acc1, sb, h1, a0, wg);
      wgmma_commit();
      wgmma_wait<0>();
      wgmma_fence_regs(acc1);
      frag_to_a<BF16, RELU, 128>(acc1, ha, P.act, P.alpha);              // h2 over h1
      // h2 for dW2 and act'(h2), over the previous tile's dz1: behind both warpgroups' dW0 of the previous tile.  (The
      // stores come before the MMA: the A registers of an MMA in flight are not read.)
      xwg_wait(kEvL0, wg);
      a_to_tile<128>(ha, h2, fr);
      float acc2[32];
      wgmma_fence();
      mma_layer2_rs<BF16>(acc2, sb, ha, a0, wg);
      wgmma_commit();
      const long long grow_lo = row0 + fr.rb;
      const float bs = Q.beta_dev[0] * Q.inv_batch * S;
      const int rows = (int)ld_shared_b32(rows_of(b));   // rows of the tile inside the batch
      mbar_wait(nz_full(b), bpar);
      if (Q.d_emb16) mbar_wait(bar_g, tk & 1);
      wgmma_wait<0>();
      wgmma_fence_regs(acc2);
      // ---- (mu, logvar) -> d(mu), d(logvar) = dO, packed as the A fragment of G2 (column e of dO is word 2 (e / 8) + h of
      // the fragment, 32 + e is 8 + 2 (e / 8) + h).  Rows past the batch end contribute nothing.
      // this thread's eps pairs: dims 8 j + 2 q (+1) of row rb + 8 h are at nzo + h * 1024 + (32 j ^ nzs) (nz_chunk with
      // chunk 2 j + q / 2), formed where they are read
      const uint32_t nzo = opaque(sb + kOffNz + b * kNzBytes + fr.rb * 128 + 8 * (fr.q & 1));
      const uint32_t nzs = opaque((((fr.rb & 7) ^ (fr.q >> 1)) << 4));
      uint32_t ao[16];
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const long long grow = grow_lo + 8 * h;
        const bool valid = fr.rb + 8 * h < rows;
        const float bsv = valid ? bs : 0.f;
        const int r = fr.rb + 8 * h;
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          const int e = 8 * j + 2 * fr.q;
          const float2 ez = ld_shared_v2f(nzo + h * 1024 + ((32 * j) ^ nzs));   // eps of dims e, e + 1
          const float nz[2] = {ez.x, ez.y};
          float g[2] = {0.f, 0.f};
          if (valid) {
            if (Q.d_emb16) unpack2<BF16>(ld_shared_b32(gbuf + 4 * (r * 16 + e / 2)), g[0], g[1]);   // [128 rows][16 pairs]
            else {
              const float2 g2 = *reinterpret_cast<const float2*>(Q.d_emb + grow * Q.ldd + f * 32 + e);
              g[0] = g2.x * S; g[1] = g2.y * S;
            }
          }
          float dm[2], dl[2];
#pragma unroll
          for (int k = 0; k < 2; ++k) {
            const float mu = acc2[4 * j + 2 * h + k], lv = acc2[4 * (j + 4) + 2 * h + k];
            const float sgm = expf(0.5f * lv);
            dm[k] = fmaf(bsv, mu, g[k]);
            dl[k] = valid ? fmaf(g[k] * nz[k], 0.5f * sgm, bsv * 0.5f * (sgm * sgm - 1.f)) : 0.f;
          }
          ao[2 * j + h] = pack2<BF16>(dm[0], dm[1]);
          ao[8 + 2 * j + h] = pack2<BF16>(dl[0], dl[1]);
        }
      }
      if (Q.d_emb16) warp_arrive(g_empty);   // this warp's d_emb16 rows are read: the producer may load the next tile's
      // dO for dW2 / db2.  The previous tile's dW2 / db2 of both warpgroups retired before its kEvDZ1 hand-off.
      a_to_tile<64>(ao, dO, fr);
      xwg_arrive(kEvDO, wg);               // this warpgroup's rows of h1, h2, dO, [pe|1] are stored; its d_emb16 rows read
      // ---- layer 2 backward: G2 = dO W2^T (own rows, A from registers) | dW2 += h2^T dO; db2 += dO^T [pe|1]
      float accd[64];
      wgmma_fence();
#pragma unroll
      for (int kk = 0; kk < EO / 16; ++kk) {
        const uint32_t a[4] = {ao[4 * kk], ao[4 * kk + 1], ao[4 * kk + 2], ao[4 * kk + 3]};
        wgmma_m64n128k16_rs<BF16, 0>(accd, a, gmma_desc(sb + kOffW2 + kk * 32, 16, 1024), kk > 0 ? 1u : 0u);
      }
      wgmma_commit();
      xwg_wait(kEvDO, wg);                 // dW2 / db2 read both warpgroups' rows of h2, dO and [pe|1]
      {
        const uint32_t h2o = opaque(h2), dOo = opaque(dO), a0o = opaque(a0), wacc = ld_shared_b32(wacc_of(b));
        wgmma_fence();
#pragma unroll
        for (int kk = 0; kk < TM / 16; ++kk)
          wgmma_m64n64k16<BF16, 1, 1>(accW2, desc_act_t_as_a(h2o, wg, kk), desc_act_as_b(dOo, kk), kk > 0 ? 1u : wacc);
        // (both warpgroups run the small db2 contraction -- uniform issue keeps the MMAs unserialised; warpgroup 0 stores it)
#pragma unroll
        for (int kk = 0; kk < TM / 16; ++kk)
          wgmma_m64n16k16<BF16, 1, 1>(accB2, desc_act_t_as_a(dOo, 0, kk), desc_a0_as_b(a0o, kk), kk > 0 ? 1u : wacc);
      }
      wgmma_commit();
      wgmma_wait<1>();
      wgmma_fence_regs(accd);
      // ---- dz2 = G2 * act'(h2), while dW2 / db2 run -> the dz2 tile (the previous tile's dW1 / db1 of both warpgroups
      // retired before its kEvDZ1 hand-off)
      {
        uint32_t az[32];
        frag_dgrad_to_a<BF16, RELU>(accd, h2, az, fr, P.act, P.alpha);
        a_to_tile<128>(az, dz2, fr);
      }
      xwg_arrive(kEvDZ2, wg);
      // ---- layer 1 backward: G1 = dz2 W1^T (own rows) | dW1 += h1^T dz2; db1 += dz2^T [pe|1]
      // G1 reads dz2 from the tile, behind a barrier of this warpgroup only.  As a register A fragment it would hold 32
      // registers through the issue of dW1 / db1, next to G1's accumulator and the weight gradients: more than 255.
      float accg[64];
      wg_publish(wg);
      wgmma_fence();
#pragma unroll
      for (int kk = 0; kk < HID / 16; ++kk)
        wgmma_m64n128k16<BF16, 0, 0>(accg, desc_act_as_a(dz2, wg, kk),
                                     gmma_desc(sb + kOffW1 + (kk >> 2) * kPanel + (kk & 3) * 32, 16, 1024), kk > 0 ? 1u : 0u);
      wgmma_commit();
      xwg_wait(kEvDZ2, wg);                // dW1 / db1 read both warpgroups' rows of dz2
      {
        const uint32_t h1o = opaque(h1), dz2o = opaque(dz2), a0o = opaque(a0), wacc = ld_shared_b32(wacc_of(b));
        wgmma_fence();
#pragma unroll
        for (int kk = 0; kk < TM / 16; ++kk)
          wgmma_m64n128k16<BF16, 1, 1>(accW1, desc_act_t_as_a(h1o, wg, kk), desc_act_as_b(dz2o, kk), kk > 0 ? 1u : wacc);
#pragma unroll
        for (int kk = 0; kk < TM / 16; ++kk)
          wgmma_m64n16k16<BF16, 1, 1>(accB1, desc_act_t_as_a(dz2o, wg, kk), desc_a0_as_b(a0o, kk), kk > 0 ? 1u : wacc);
      }
      wgmma_commit();
      wgmma_wait<1>();                     // G1, and dW2 / db2 before it
      wgmma_fence_regs(accg); wgmma_fence_regs(accW2); wgmma_fence_regs(accB2);
      xwg_arrive(kEvDW2, wg);              // this warpgroup's dW2 (it read all of h2) is done
      // ---- dz1 = G1 * act'(h1) -> the h2 buffer, while dW1 / db1 run (they read h1, dz2, [pe|1])
      uint32_t az[32];
      frag_dgrad_to_a<BF16, RELU>(accg, h1, az, fr, P.act, P.alpha);
      xwg_wait(kEvDW2, wg);                // dz1 is written over h2 only after every dW2 of the tile
      a_to_tile<128>(az, h2, fr);
      wgmma_wait<0>();
      wgmma_fence_regs(accW1); wgmma_fence_regs(accB1);
      // dz1 stored, and this warpgroup's dW1 / db1 (they read all of h1, dz2) done: h1, dz2 and dO may be rewritten
      xwg_arrive(kEvDZ1, wg);
      xwg_wait(kEvDZ1, wg);                // dW0 reads both warpgroups' rows of dz1
      // ---- layer 0 backward: [dW0;db0]^T += dz1^T [pe|1], retired by the next tile's layer-0 wait (or after the loop)
      {
        const uint32_t h2o = opaque(h2), a0o = opaque(a0), wacc = ld_shared_b32(wacc_of(b));
        wgmma_fence();
#pragma unroll
        for (int kk = 0; kk < TM / 16; ++kk)
          wgmma_m64n16k16<BF16, 1, 1>(accW0, desc_act_t_as_a(h2o, wg, kk), desc_a0_as_b(a0o, kk), kk > 0 ? 1u : wacc);
      }
      wgmma_commit();
    }
    wgmma_wait<0>();
    wgmma_fence_regs(accW0);
    warp_arrive(w_empty);                  // this warp's MMAs of the feature (the weights' last readers) retired
    const bool ran = (long long)sched_here(F).slot * TM < P.n;
    if (ran) warp_arrive(slot_empty((tk - 1) & 1));   // the last tile's dW0 retired
    // ================= flush this (feature, slot)'s weight-gradient partials (scaled back by 1/S)
    float* part = Q.part + (long long)sched_here(F).slot * Q.split_stride;
    const int w_in = P.fdim[f] * P.nfreq;
    const float invS = 1.f / __uint_as_float(opaque(__float_as_uint(S)));
    auto out = [&](float v) { return ran ? v * invS : 0.f; };
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int m = fr.rb + 8 * h;                       // this thread's rows of the warpgroup-owned accumulators
#pragma unroll
      for (int j = 0; j < 16; ++j)                       // dW1[h1 = m][h2 = 8 j + 2 q ..]
        *reinterpret_cast<float2*>(part + Q.w1_off[f] + (long long)m * HID + 8 * j + 2 * fr.q) =
            make_float2(out(accW1[4 * j + 2 * h]), out(accW1[4 * j + 2 * h + 1]));
#pragma unroll
      for (int j = 0; j < 8; ++j)                        // dW2[h2 = m][o = 8 j + 2 q ..]
        *reinterpret_cast<float2*>(part + Q.w2_off[f] + (long long)m * EO + 8 * j + 2 * fr.q) =
            make_float2(out(accW2[4 * j + 2 * h]), out(accW2[4 * j + 2 * h + 1]));
      // dW0[k][h1 = m] (k < w_in) and db0[m] = column w_in of dW0p^T; db1[h2 = m], db2[o = m] = column w_in
#pragma unroll
      for (int j = 0; j < 2; ++j) {
#pragma unroll
        for (int k = 0; k < 2; ++k) {
          const int col = 8 * j + 2 * fr.q + k;
          const float v0 = out(accW0[4 * j + 2 * h + k]);
          if (col < w_in) part[Q.w0_off[f] + (long long)col * HID + m] = v0;
          else if (col == w_in) {
            part[Q.b0_off[f] + m] = v0;
            part[P.b1_off[f] + m] = out(accB1[4 * j + 2 * h + k]);
            if (wg == 0) part[P.b2_off[f] + m] = out(accB2[4 * j + 2 * h + k]);
          }
        }
      }
    }
  }
}

// ----------------------------------------------------------------------------------------------------
// fp32 master parameters -> packed 16-bit per-feature weights [W0p | W1 | W2 | Bb1 | Bb2]
// (bias of layer 0 folded into W0p row w_in; b1 / b2 in row w_in of the bias carriers)
// ----------------------------------------------------------------------------------------------------
template <bool BF16>
__global__ void dib_enc_pack_weights_kernel(const float* __restrict__ params, const long long* __restrict__ w0_off,
                                            const long long* __restrict__ b0_off, const long long* __restrict__ w1_off,
                                            const long long* __restrict__ b1_off, const long long* __restrict__ w2_off,
                                            const long long* __restrict__ b2_off, const int* __restrict__ fdim, int nfreq,
                                            float logvar_offset, uint16_t* __restrict__ out, float* __restrict__ zero, long long zero_n) {
  const int f = blockIdx.y;
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  {   // the KL partial-sum table of the forward kernel that follows is cleared here (one launch instead of a memset node)
    const long long z = ((long long)f * gridDim.x + blockIdx.x) * blockDim.x + threadIdx.x;
    if (z < zero_n) zero[z] = 0.f;
  }
  if (i >= kPackElems) return;
  const int idx = i, w_in = fdim[f] * nfreq;
  float v;
  if (i < kW0Elems) {
    const int k = i / HID, n = i - k * HID;
    v = k < w_in ? params[w0_off[f] + (long long)k * HID + n] : (k == w_in ? params[b0_off[f] + n] : 0.f);
  } else if ((i -= kW0Elems) < kW1Elems) {
    v = params[w1_off[f] + i];
  } else if ((i -= kW1Elems) < kW2Elems) {
    v = params[w2_off[f] + i];
  } else if ((i -= kW2Elems) < kB1Elems) {
    const int k = i / HID, n = i - k * HID;
    v = k == w_in ? params[b1_off[f] + n] : 0.f;
  } else {
    i -= kB1Elems;
    const int k = i / EO, n = i - k * EO;
    v = k == w_in ? params[b2_off[f] + n] + (n >= EO / 2 ? logvar_offset : 0.f) : 0.f;
  }
  // saturating like every activation operand: a weight beyond fp16's 65 504 packs as +-65 504, not inf
  out[(long long)f * kPackElems + idx] = (uint16_t)(pack2<BF16>(v, 0.f) & 0xffffu);
}

typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                  const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                  CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
EncodeTiledFn encode_fn2() {
  static EncodeTiledFn fn = nullptr;
  if (!fn) {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) == cudaSuccess &&
        q == cudaDriverEntryPointSuccess)
      fn = reinterpret_cast<EncodeTiledFn>(p);
  }
  return fn;
}

// [rows x cols] 16-bit matrix per feature -> 3D map (col, row, feature), box 64 cols x rows x 1, SWIZZLE_128B
bool make_wmap(CUtensorMap* m, const uint16_t* base, int cols, int rows, int nfeat, bool bf16) {
  cuuint64_t dims[3] = {(cuuint64_t)cols, (cuuint64_t)rows, (cuuint64_t)nfeat};
  cuuint64_t strides[2] = {(cuuint64_t)cols * 2, (cuuint64_t)kPackElems * 2};
  cuuint32_t box[3] = {64, (cuuint32_t)rows, 1};
  cuuint32_t es[3] = {1, 1, 1};
  return encode_fn2()(m, bf16 ? CU_TENSOR_MAP_DATA_TYPE_BFLOAT16 : CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 3,
                      const_cast<uint16_t*>(base), dims, strides, box, es, CU_TENSOR_MAP_INTERLEAVE_NONE,
                      CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                      CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) == CUDA_SUCCESS;
}

// d_emb16 [n rows, pitch ld] 16-bit, columns [0, cols) -> 2D map, box 32 cols x 128 rows (one feature's block of a tile),
// no swizzle; rows past n are filled with zeros
bool make_gmap(CUtensorMap* m, const void* base, int cols, long long n, int ld, bool bf16) {
  cuuint64_t dims[2] = {(cuuint64_t)cols, (cuuint64_t)n};
  cuuint64_t strides[1] = {(cuuint64_t)ld * 2};
  cuuint32_t box[2] = {32, TM};
  cuuint32_t es[2] = {1, 1};
  return encode_fn2()(m, bf16 ? CU_TENSOR_MAP_DATA_TYPE_BFLOAT16 : CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 2,
                      const_cast<void*>(base), dims, strides, box, es, CU_TENSOR_MAP_INTERLEAVE_NONE,
                      CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_NONE,
                      CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) == CUDA_SUCCESS;
}

bool make_all_maps(WeightMaps* m, const void* packed, int F, bool bf16) {
  const uint16_t* pk = static_cast<const uint16_t*>(packed);
  return make_wmap(&m->w0, pk, HID, K0, F, bf16) && make_wmap(&m->w1, pk + kW0Elems, HID, HID, F, bf16) &&
         make_wmap(&m->w2, pk + kW0Elems + kW1Elems, EO, HID, F, bf16) &&
         make_wmap(&m->b1, pk + kW0Elems + kW1Elems + kW2Elems, HID, K0, F, bf16) &&
         make_wmap(&m->b2, pk + kW0Elems + kW1Elems + kW2Elems + kB1Elems, EO, K0, F, bf16);
}

void fill_params(EncFusedParams& P, const DibEncFusedDesc& d, const DibEncFusedIO& io) {
  P.x = io.x; P.ldx = io.ldx; P.x_off = d.x_off; P.fdim = d.fdim; P.nfreq = d.nfreq; P.params = io.params;
  P.b1_off = d.b1_off; P.b2_off = d.b2_off; P.eps = io.eps; P.seed = io.seed; P.step = io.step; P.step_dev = io.step_dev;
  P.sample_offset = io.sample_offset; P.emb = io.emb; P.ldemb = io.ldemb; P.user_emb = io.user_emb;
  P.kl_part = io.kl_part; P.kl_stride = io.kl_stride; P.F = d.F; P.n = io.n; P.act = d.act; P.alpha = d.alpha;
  P.round_emb = 1; P.emb16 = static_cast<uint16_t*>(io.emb16); P.ldemb16 = io.ldemb16;
}

template <typename K, typename... A>
cudaError_t launch_fused(K kern, int threads, int smem, int grid, cudaStream_t st, const A&... args) {
  cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
  if (e != cudaSuccess) return e;
  kern<<<grid, threads, smem, st>>>(args...);
  dib_note_launch();
  return cudaGetLastError();
}

}  // namespace

size_t dib_enc_fused_pack_bytes(int F) { return (size_t)F * kPackElems * 2; }
long long dib_enc_fused_pack_zero_capacity(int F) { return (long long)DIB_CEIL_DIV(kPackElems, 256) * 256 * F; }   // floats the pack kernel can also clear
int dib_enc_fused_fwd_ctas_per_sm() { return 2; }

cudaError_t dib_enc_fused_pack(const DibEncFusedDesc& d, const float* params, void* packed, float* zero, long long zero_n, cudaStream_t st) {
  dim3 grid(DIB_CEIL_DIV(kPackElems, 256), d.F);
  if (zero_n > (long long)grid.x * grid.y * 256) return cudaErrorInvalidValue;
  if (d.bf16)
    dib_enc_pack_weights_kernel<true><<<grid, 256, 0, st>>>(params, d.w0_off, d.b0_off, d.w1_off, d.b1_off, d.w2_off,
                                                           d.b2_off, d.fdim, d.nfreq, d.logvar_offset, static_cast<uint16_t*>(packed), zero, zero_n);
  else
    dib_enc_pack_weights_kernel<false><<<grid, 256, 0, st>>>(params, d.w0_off, d.b0_off, d.w1_off, d.b1_off, d.w2_off,
                                                            d.b2_off, d.fdim, d.nfreq, d.logvar_offset, static_cast<uint16_t*>(packed), zero, zero_n);
  dib_note_launch();
  return cudaGetLastError();
}

cudaError_t dib_enc_fused_forward(const DibEncFusedDesc& d, const DibEncFusedIO& io, cudaStream_t st) {
  if (!encode_fn2()) return cudaErrorNotSupported;
  WeightMaps m;
  if (!make_all_maps(&m, io.packed, d.F, d.bf16)) return cudaErrorInvalidValue;
  EncFusedParams P;
  fill_params(P, d, io);
  constexpr int smem = kOffFwdEnd + 128 + 1024;
  const bool relu = d.act == DIB_ACT_RELU;
  if (d.bf16) return relu ? launch_fused(dib_enc_fused_fwd_kernel<true, true>, kThreads, smem, d.grid, st, m, P)
                          : launch_fused(dib_enc_fused_fwd_kernel<true, false>, kThreads, smem, d.grid, st, m, P);
  return relu ? launch_fused(dib_enc_fused_fwd_kernel<false, true>, kThreads, smem, d.grid, st, m, P)
              : launch_fused(dib_enc_fused_fwd_kernel<false, false>, kThreads, smem, d.grid, st, m, P);
}

cudaError_t dib_enc_fused_backward(const DibEncFusedDesc& d, const DibEncFusedIO& io, const DibEncFusedBwdIO& b,
                                   cudaStream_t st) {
  if (!encode_fn2()) return cudaErrorNotSupported;
  WeightMaps m;
  if (!make_all_maps(&m, io.packed, d.F, d.bf16)) return cudaErrorInvalidValue;
  EncFusedBwdParams Q;
  fill_params(Q.f, d, io);
  Q.f.round_emb = 0;
  Q.d_emb16 = static_cast<const uint16_t*>(b.d_emb16);
  CUtensorMap gmap = {};                  // unused without d_emb16
  if (b.d_emb16 && !make_gmap(&gmap, b.d_emb16, d.F * 32, io.n, b.ldd16, d.bf16)) return cudaErrorInvalidValue;
  Q.d_emb = b.d_emb; Q.ldd = b.ldd; Q.beta_dev = b.beta_dev; Q.inv_batch = b.inv_batch; Q.gscale = b.gscale;
  Q.part = b.part; Q.split_stride = b.split_stride;
  Q.w0_off = d.w0_off; Q.b0_off = d.b0_off; Q.w1_off = d.w1_off; Q.w2_off = d.w2_off;
  constexpr int smem = kOffBwdEnd + 128 + 1024;
  const bool relu = d.act == DIB_ACT_RELU;
  if (d.bf16) return relu ? launch_fused(dib_enc_fused_bwd_kernel<true, true>, kBwdThreads, smem, d.grid, st, m, gmap, Q)
                          : launch_fused(dib_enc_fused_bwd_kernel<true, false>, kBwdThreads, smem, d.grid, st, m, gmap, Q);
  return relu ? launch_fused(dib_enc_fused_bwd_kernel<false, true>, kBwdThreads, smem, d.grid, st, m, gmap, Q)
              : launch_fused(dib_enc_fused_bwd_kernel<false, false>, kBwdThreads, smem, d.grid, st, m, gmap, Q);
}
