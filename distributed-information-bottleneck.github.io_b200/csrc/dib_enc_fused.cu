// dib_enc_fused.cu -- the fused per-feature encoder kernels of the tensor-core mode (sm_90a).
//
// One persistent CTA works on ONE feature at a time: the feature's encoder weights (positional-encoding layer incl. its
// bias row, 128x128 hidden layer, 128x64 (mu|logvar) layer) are TMA-staged into shared memory once and reused for every
// 128-sample tile of that feature.  Per tile the whole chain of models.py:101-112
//     x column -> positional encoding -> Dense(128,act) -> Dense(128,act) -> Dense(2E) -> split (mu, logvar)
//     -> u = mu + exp(logvar/2) eps -> KL partial sums -> emb[:, f*E:(f+1)*E]
// runs on chip: the three contractions are wgmma instructions (16-bit operands with an 11-bit significand = TF32's, fp32
// accumulation in registers), the activations travel registers -> shared memory (as the next MMA's swizzled A operand)
// and never touch HBM.  Only x (4 B/sample/feature) is read and emb is written.
//
// Two warpgroups per CTA; warpgroup g owns rows [64 g, 64 g + 64) of a tile (wgmma M = 64).  Every contraction whose
// reduction runs over the hidden features (forward, dgrad) reads only the warpgroup's own rows, so the two warpgroups
// proceed independently; the weight-gradient contractions of the backward reduce over all 128 samples of the tile and
// meet at CTA barriers.
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
constexpr int kOffA0 = kOffBb2 + K0 * 128;         // 2 KB : Bb2 = 1 panel x 16 rows x 128 B
constexpr int kOffH1 = kOffA0 + 2 * TM * 16 + 2048;// 4 KB : A0 = [2 k-halves][128 rows][16 B] (no swizzle); +2 KB keeps 1024-alignment
constexpr int kOffFwdEnd = kOffH1 + 2 * kPanel;    // forward: h2 overwrites h1 (the layer-1 MMA that read it has retired)
// backward-only tiles
constexpr int kOffH2 = kOffH1 + 2 * kPanel;        // h2, later dz1
constexpr int kOffDO = kOffH2 + 2 * kPanel;        // [128 x 64] d(mu | logvar), one panel
constexpr int kOffDZ2 = kOffDO + kPanel;           // [128 x 128]
constexpr int kOffBwdEnd = kOffDZ2 + 2 * kPanel;
static_assert(kOffH1 % 1024 == 0 && kOffDZ2 % 1024 == 0, "operand tiles must be 1024-byte aligned");

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

// address of the 16-byte chunk holding columns [8c, 8c+8) of row r in a [128 x 64k] swizzled tile
__device__ __forceinline__ uint32_t tile_chunk_addr(uint32_t tile, int r, int col) {
  const int panel = col >> 6, c = (col & 63) >> 3;
  return tile + panel * kPanel + r * 128 + ((c ^ (r & 7)) << 4);
}

// Position of this thread's accumulator elements in the tile: rows rb and rb + 8, columns 8 j + 2 q (+1).
struct Frag {
  int rb, q;
};
__device__ __forceinline__ Frag frag_of(int tid) {
  const int wg = tid >> 7, wq = (tid >> 5) & 3, lane = tid & 31;
  return Frag{64 * wg + 16 * wq + (lane >> 2), lane & 3};
}

// accumulator of a 64 x N tile -> activation -> 16-bit -> the swizzled shared tile (the next MMA's A operand).  The bias is
// already in the accumulator.  Each quad of lanes writes one 16-byte chunk of a row: conflict-free under the swizzle.
template <bool BF16, bool RELU, int N>
__device__ __forceinline__ void frag_to_tile(const float (&d)[N / 2], uint32_t tile, Frag fr, int act, float alpha) {
#pragma unroll
  for (int j = 0; j < N / 8; ++j) {
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const float v0 = d[4 * j + 2 * h], v1 = d[4 * j + 2 * h + 1];
      const uint32_t w = RELU ? pack2_relu<BF16>(v0, v1) : pack2<BF16>(dib_act16(act, v0, alpha), dib_act16(act, v1, alpha));
      st_shared_b32(tile_chunk_addr(tile, fr.rb + 8 * h, 8 * j) + 4 * fr.q, w);
    }
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

// gradient accumulator (64 x 128) * act'(h) -> 16-bit -> shared tile `dtile`; h is read back from the shared tile `htile`
// that the recomputed forward wrote (relu: as a packed comparison, other activations through act'(h)).  dtile may be htile.
template <bool BF16, bool RELU>
__device__ __forceinline__ void frag_dgrad_to_tile(const float (&d)[64], uint32_t htile, uint32_t dtile, Frag fr, int act,
                                                   float alpha) {
#pragma unroll
  for (int j = 0; j < 16; ++j) {
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const uint32_t off = tile_chunk_addr(0u, fr.rb + 8 * h, 8 * j) + 4 * fr.q;
      const uint32_t hv = ld_shared_b32(htile + off);
      const float g0 = d[4 * j + 2 * h], g1 = d[4 * j + 2 * h + 1];
      uint32_t o;
      if constexpr (RELU) {
        o = relu_gate2<BF16>(pack2<BF16>(g0, g1), hv);
      } else {
        float h0, h1;
        unpack2<BF16>(hv, h0, h1);
        o = pack2<BF16>(g0 * dib_act_grad(act, h0, alpha), g1 * dib_act_grad(act, h1, alpha));
      }
      st_shared_b32(dtile + off, o);
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
__device__ __forceinline__ void load_x(const float* xrow, int d, float (&xv)[kMaxFeatDim]) {
#pragma unroll
  for (int j = 0; j < kMaxFeatDim; ++j) xv[j] = (xrow && j < d) ? xrow[j] : 0.f;
}
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
template <bool BF16>
__device__ __forceinline__ void stage_a0(const EncFusedParams& P, uint32_t a0, int tid, long long row0, int d, int xo) {
  const int ar = 64 * (tid >> 7) + (tid & 63), khalf = (tid >> 6) & 1;
  const long long grow = row0 + ar;
  float xv[kMaxFeatDim];
  load_x(grow < P.n ? P.x + grow * P.ldx + xo : nullptr, d, xv);
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
// activation tile as A (K-major): k step kk of 16 features
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
template <bool BF16>
__device__ __forceinline__ void mma_layer1(float (&d)[64], uint32_t sb, uint32_t h1, uint32_t a0, int wg) {
  wgmma_m64n128k16<BF16, 0, 1>(d, desc_a0_as_a(a0, wg), gmma_desc(sb + kOffBb1, K0 * 128, 1024), 0u);
#pragma unroll
  for (int kk = 0; kk < HID / 16; ++kk)
    wgmma_m64n128k16<BF16, 0, 1>(d, desc_act_as_a(h1, wg, kk), gmma_desc(sb + kOffW1 + kk * 2048, kPanel, 1024), 1u);
}
template <bool BF16>
__device__ __forceinline__ void mma_layer2(float (&d)[32], uint32_t sb, uint32_t h2, uint32_t a0, int wg) {
  wgmma_m64n64k16<BF16, 0, 1>(d, desc_a0_as_a(a0, wg), gmma_desc(sb + kOffBb2, K0 * 128, 1024), 0u);
#pragma unroll
  for (int kk = 0; kk < HID / 16; ++kk)
    wgmma_m64n64k16<BF16, 0, 1>(d, desc_act_as_a(h2, wg, kk), gmma_desc(sb + kOffW2 + kk * 2048, kPanel, 1024), 1u);
}

// shared tile written by this warpgroup -> visible to its MMAs
__device__ __forceinline__ void wg_publish(int wg) {
  fence_proxy_async_smem();
  named_bar_sync(1 + wg, 128);
}
// ... to the MMAs of both warpgroups
__device__ __forceinline__ void cta_publish() {
  fence_proxy_async_smem();
  __syncthreads();
}

// feature / tile assignment of a persistent CTA: with at least as many CTAs as features, CTA c serves feature c % F and
// its tiles slot, slot + nslots, ...; otherwise it walks features c, c + G, ... with all of their tiles
struct Sched { int f_first, f_step, slot, nslots; };
__device__ __forceinline__ Sched sched_of(int c, int G, int F) {
  if (G >= F) { const int f0 = c % F; return Sched{f0, F * G, c / F, (G - f0 + F - 1) / F}; }
  return Sched{c, G, 0, 1};
}

// ====================================================================================================
// forward: x -> emb, KL partial sums.  96 KB of shared memory -> two CTAs per SM, so one CTA's epilogue overlaps the
// other's MMAs.
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
  const uint32_t a0 = sb + kOffA0, hbuf = sb + kOffH1;

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
    float kl_acc = 0.f;
    mbar_wait(bar_w, fit & 1);
    for (int t = s.slot; t < ntiles; t += s.nslots) {
      const long long row0 = (long long)t * TM;
      stage_a0<BF16>(P, a0, tid, row0, d, xo);
      wg_publish(wg);
      float acc[64];
      wgmma_fence();
      mma_layer0<BF16>(acc, sb, a0, wg);
      wgmma_commit();
      wgmma_wait<0>();
      wgmma_fence_regs(acc);
      frag_to_tile<BF16, RELU, 128>(acc, hbuf, fr, P.act, P.alpha);
      wg_publish(wg);
      wgmma_fence();
      mma_layer1<BF16>(acc, sb, hbuf, a0, wg);
      wgmma_commit();
      wgmma_wait<0>();
      wgmma_fence_regs(acc);
      frag_to_tile<BF16, RELU, 128>(acc, hbuf, fr, P.act, P.alpha);      // h2 over h1
      wg_publish(wg);
      float acc2[32];
      wgmma_fence();
      mma_layer2<BF16>(acc2, sb, hbuf, a0, wg);
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
// warpgroup g owns rows [64 g, 64 g + 64) of dW1, dW2 (and of dW0^T, db1); warpgroup 0 stores db2.  176 KB of shared
// memory: one CTA per SM.
// ====================================================================================================
struct EncFusedBwdParams {
  EncFusedParams f;
  const float* d_emb; int ldd;              // [n, ldd] gradient w.r.t. emb (already scaled by 1/B_global)
  const uint16_t* d_emb16; int ldd16;       // or: 16-bit gradient already multiplied by the loss scale S
  const float* beta_dev; float inv_batch; float gscale;
  float* part; long long split_stride;      // weight-gradient partials [slot][P]
  const long long* w0_off; const long long* b0_off; const long long* w1_off; const long long* w2_off;
};

template <bool BF16, bool RELU>
__global__ void __launch_bounds__(kThreads, 1)
dib_enc_fused_bwd_kernel(const __grid_constant__ WeightMaps maps, const EncFusedBwdParams Q) {
  const EncFusedParams& P = Q.f;
  extern __shared__ uint8_t smem_raw[];
  const uint32_t sb = (smem_u32(smem_raw) + 1023u) & ~1023u;
  const uint32_t bar_w = sb + kOffBwdEnd;

  const int tid = threadIdx.x, lane = tid & 31, wg = tid >> 7;
  const Frag fr = frag_of(tid);
  const int F = P.F;
  const int ntiles = (int)((P.n + TM - 1) / TM);
  const unsigned int nstep = P.step + (P.step_dev ? P.step_dev[0] : 0u);
  const uint32_t a0 = sb + kOffA0, h1 = sb + kOffH1, h2 = sb + kOffH2, dO = sb + kOffDO, dz2 = sb + kOffDZ2;
  const float S = Q.gscale, invS = 1.f / Q.gscale;

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
    const float bs = Q.beta_dev[0] * Q.inv_batch * S;
    float accW1[64], accW2[32], accW0[8], accB1[8], accB2[8];
#pragma unroll
    for (int i = 0; i < 64; ++i) accW1[i] = 0.f;
#pragma unroll
    for (int i = 0; i < 32; ++i) accW2[i] = 0.f;
#pragma unroll
    for (int i = 0; i < 8; ++i) { accW0[i] = 0.f; accB1[i] = 0.f; accB2[i] = 0.f; }
    mbar_wait(bar_w, fit & 1);
    for (int t = s.slot; t < ntiles; t += s.nslots) {
      const long long row0 = (long long)t * TM;
      // ---- recompute the forward of this warpgroup's rows
      stage_a0<BF16>(P, a0, tid, row0, d, xo);
      wg_publish(wg);
      float acc[64];
      wgmma_fence();
      mma_layer0<BF16>(acc, sb, a0, wg);
      wgmma_commit();
      wgmma_wait<0>();
      wgmma_fence_regs(acc);
      frag_to_tile<BF16, RELU, 128>(acc, h1, fr, P.act, P.alpha);
      wg_publish(wg);
      wgmma_fence();
      mma_layer1<BF16>(acc, sb, h1, a0, wg);
      wgmma_commit();
      wgmma_wait<0>();
      wgmma_fence_regs(acc);
      frag_to_tile<BF16, RELU, 128>(acc, h2, fr, P.act, P.alpha);
      wg_publish(wg);
      float acc2[32];
      wgmma_fence();
      mma_layer2<BF16>(acc2, sb, h2, a0, wg);
      wgmma_commit();
      const long long grow_lo = row0 + fr.rb;
      float nz[4][2][2];
#pragma unroll
      for (int j = 0; j < 4; ++j) noise_pair(P, nstep, grow_lo, f, j, fr.q, lane, nz[j]);
      wgmma_wait<0>();
      wgmma_fence_regs(acc2);
      // ---- (mu, logvar) -> d(mu), d(logvar) -> dO tile.  Rows past the batch end contribute nothing.
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const long long grow = grow_lo + 8 * h;
        const bool valid = grow < P.n;
        const float bsv = valid ? bs : 0.f;
        const int r = fr.rb + 8 * h;
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          const int e = 8 * j + 2 * fr.q;
          float g[2] = {0.f, 0.f};
          if (valid) {
            if (Q.d_emb16) unpack2<BF16>(*reinterpret_cast<const uint32_t*>(Q.d_emb16 + grow * Q.ldd16 + f * 32 + e), g[0], g[1]);
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
            dl[k] = valid ? fmaf(g[k] * nz[j][h][k], 0.5f * sgm, bsv * 0.5f * (sgm * sgm - 1.f)) : 0.f;
          }
          st_shared_b32(tile_chunk_addr(dO, r, e) + 4 * fr.q, pack2<BF16>(dm[0], dm[1]));
          st_shared_b32(tile_chunk_addr(dO, r, 32 + e) + 4 * fr.q, pack2<BF16>(dl[0], dl[1]));
        }
      }
      cta_publish();                       // dO, h2, h1, [pe|1] of all 128 rows
      // ---- layer 2 backward: G2 = dO W2^T (own rows); dW2 += h2^T dO; db2 += dO^T [pe|1]
      wgmma_fence();
#pragma unroll
      for (int kk = 0; kk < EO / 16; ++kk)
        wgmma_m64n128k16<BF16, 0, 0>(acc, gmma_desc(dO + wg * 64 * 128 + kk * 32, 16, 1024),
                                     gmma_desc(sb + kOffW2 + kk * 32, 16, 1024), kk > 0 ? 1u : 0u);
#pragma unroll
      for (int kk = 0; kk < TM / 16; ++kk)
        wgmma_m64n64k16<BF16, 1, 1>(accW2, desc_act_t_as_a(h2, wg, kk), desc_act_as_b(dO, kk), 1u);
      // (both warpgroups run the small db2 contraction -- uniform issue keeps the MMAs unserialised; warpgroup 0 stores it)
#pragma unroll
      for (int kk = 0; kk < TM / 16; ++kk)
        wgmma_m64n16k16<BF16, 1, 1>(accB2, desc_act_t_as_a(dO, 0, kk), desc_a0_as_b(a0, kk), 1u);
      wgmma_commit();
      wgmma_wait<0>();
      wgmma_fence_regs(acc); wgmma_fence_regs(accW2); wgmma_fence_regs(accB2);
      // ---- dz2 = G2 * act'(h2)
      frag_dgrad_to_tile<BF16, RELU>(acc, h2, dz2, fr, P.act, P.alpha);
      cta_publish();
      // ---- layer 1 backward: G1 = dz2 W1^T (own rows); dW1 += h1^T dz2; db1 += dz2^T [pe|1]
      wgmma_fence();
#pragma unroll
      for (int kk = 0; kk < HID / 16; ++kk)
        wgmma_m64n128k16<BF16, 0, 0>(acc, desc_act_as_a(dz2, wg, kk),
                                     gmma_desc(sb + kOffW1 + (kk >> 2) * kPanel + (kk & 3) * 32, 16, 1024), kk > 0 ? 1u : 0u);
#pragma unroll
      for (int kk = 0; kk < TM / 16; ++kk)
        wgmma_m64n128k16<BF16, 1, 1>(accW1, desc_act_t_as_a(h1, wg, kk), desc_act_as_b(dz2, kk), 1u);
#pragma unroll
      for (int kk = 0; kk < TM / 16; ++kk)
        wgmma_m64n16k16<BF16, 1, 1>(accB1, desc_act_t_as_a(dz2, wg, kk), desc_a0_as_b(a0, kk), 1u);
      wgmma_commit();
      wgmma_wait<0>();
      wgmma_fence_regs(acc); wgmma_fence_regs(accW1); wgmma_fence_regs(accB1);
      // ---- dz1 = G1 * act'(h1) -> the h2 buffer (its last readers, the dz2 epilogue and dW2, are done)
      frag_dgrad_to_tile<BF16, RELU>(acc, h1, h2, fr, P.act, P.alpha);
      cta_publish();
      // ---- layer 0 backward: [dW0;db0]^T += dz1^T [pe|1]
      wgmma_fence();
#pragma unroll
      for (int kk = 0; kk < TM / 16; ++kk)
        wgmma_m64n16k16<BF16, 1, 1>(accW0, desc_act_t_as_a(h2, wg, kk), desc_a0_as_b(a0, kk), 1u);
      wgmma_commit();
      wgmma_wait<0>();
      wgmma_fence_regs(accW0);
      __syncthreads();                     // every MMA of this tile has read its operands: the next tile may overwrite them
    }
    // ================= flush this (feature, slot)'s weight-gradient partials (scaled back by 1/S)
    float* part = Q.part + (long long)s.slot * Q.split_stride;
    const int w_in = d * P.nfreq;
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int m = fr.rb + 8 * h;                       // this thread's rows of the warpgroup-owned accumulators
#pragma unroll
      for (int j = 0; j < 16; ++j)                       // dW1[h1 = m][h2 = 8 j + 2 q ..]
        *reinterpret_cast<float2*>(part + Q.w1_off[f] + (long long)m * HID + 8 * j + 2 * fr.q) =
            make_float2(accW1[4 * j + 2 * h] * invS, accW1[4 * j + 2 * h + 1] * invS);
#pragma unroll
      for (int j = 0; j < 8; ++j)                        // dW2[h2 = m][o = 8 j + 2 q ..]
        *reinterpret_cast<float2*>(part + Q.w2_off[f] + (long long)m * EO + 8 * j + 2 * fr.q) =
            make_float2(accW2[4 * j + 2 * h] * invS, accW2[4 * j + 2 * h + 1] * invS);
      // dW0[k][h1 = m] (k < w_in) and db0[m] = column w_in of dW0p^T; db1[h2 = m], db2[o = m] = column w_in
#pragma unroll
      for (int j = 0; j < 2; ++j) {
#pragma unroll
        for (int k = 0; k < 2; ++k) {
          const int col = 8 * j + 2 * fr.q + k;
          const float v0 = accW0[4 * j + 2 * h + k] * invS;
          if (col < w_in) part[Q.w0_off[f] + (long long)col * HID + m] = v0;
          else if (col == w_in) {
            part[Q.b0_off[f] + m] = v0;
            part[P.b1_off[f] + m] = accB1[4 * j + 2 * h + k] * invS;
            if (wg == 0) part[P.b2_off[f] + m] = accB2[4 * j + 2 * h + k] * invS;
          }
        }
      }
    }
    __syncthreads();                       // both warpgroups are done with this feature's weights
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
  uint16_t h;
  if constexpr (BF16) { __nv_bfloat16 b = __float2bfloat16_rn(v); h = *reinterpret_cast<uint16_t*>(&b); }
  else { __half b = __float2half_rn(v); h = *reinterpret_cast<uint16_t*>(&b); }
  out[(long long)f * kPackElems + idx] = h;
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

template <typename K, typename A>
cudaError_t launch_fused(K kern, int smem, int grid, const WeightMaps& m, const A& args, cudaStream_t st) {
  cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
  if (e != cudaSuccess) return e;
  kern<<<grid, kThreads, smem, st>>>(m, args);
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
  if (d.bf16) return relu ? launch_fused(dib_enc_fused_fwd_kernel<true, true>, smem, d.grid, m, P, st)
                          : launch_fused(dib_enc_fused_fwd_kernel<true, false>, smem, d.grid, m, P, st);
  return relu ? launch_fused(dib_enc_fused_fwd_kernel<false, true>, smem, d.grid, m, P, st)
              : launch_fused(dib_enc_fused_fwd_kernel<false, false>, smem, d.grid, m, P, st);
}

cudaError_t dib_enc_fused_backward(const DibEncFusedDesc& d, const DibEncFusedIO& io, const DibEncFusedBwdIO& b,
                                   cudaStream_t st) {
  if (!encode_fn2()) return cudaErrorNotSupported;
  WeightMaps m;
  if (!make_all_maps(&m, io.packed, d.F, d.bf16)) return cudaErrorInvalidValue;
  EncFusedBwdParams Q;
  fill_params(Q.f, d, io);
  Q.f.round_emb = 0;
  Q.d_emb16 = static_cast<const uint16_t*>(b.d_emb16); Q.ldd16 = b.ldd16;
  Q.d_emb = b.d_emb; Q.ldd = b.ldd; Q.beta_dev = b.beta_dev; Q.inv_batch = b.inv_batch; Q.gscale = b.gscale;
  Q.part = b.part; Q.split_stride = b.split_stride;
  Q.w0_off = d.w0_off; Q.b0_off = d.b0_off; Q.w1_off = d.w1_off; Q.w2_off = d.w2_off;
  constexpr int smem = kOffBwdEnd + 128 + 1024;
  const bool relu = d.act == DIB_ACT_RELU;
  if (d.bf16) return relu ? launch_fused(dib_enc_fused_bwd_kernel<true, true>, smem, d.grid, m, Q, st)
                          : launch_fused(dib_enc_fused_bwd_kernel<true, false>, smem, d.grid, m, Q, st);
  return relu ? launch_fused(dib_enc_fused_bwd_kernel<false, true>, smem, d.grid, m, Q, st)
              : launch_fused(dib_enc_fused_bwd_kernel<false, false>, smem, d.grid, m, Q, st);
}
