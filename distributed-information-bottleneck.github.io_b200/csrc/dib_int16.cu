// dib_int16.cu -- the integration network (models.py:81-84,122) in the tensor-core mode: 16-bit activations in HBM
// (emb, g_k, dz_k as fp16 -> half the traffic of the fp32 layout), wgmma on 16-bit operands with fp32 accumulation.
//
//   * dib_int16_gemm_kernel<MODE>: TMA-fed, mbarrier-pipelined 128 x 128 tile GEMM (K step 64 = one 128-byte swizzle
//     span) with fused epilogues:  FWD  g = act(A W + b) -> fp16;  DGRAD  dz_in = (dz W^T) * act'(g_in) -> fp16 and the
//     column sums of dz_in (bias gradient of the layer below);  WGRAD  dW = g^T dz over a batch slice -> fp32 split partial
//     (scaled back by 1/S).
//   * dib_int16_head_kernel: the narrow output layer (out <= 16) fused with everything around it -- logits, compiled
//     loss + accuracy, d loss / d logits, the dgrad into the last hidden layer (incl. its act') and the output layer's
//     own weight/bias gradients -- one pass over the last hidden activation.
//   * dib_int16_fwd2_kernel: the last two 256-wide hidden layers and the single-output head of models with out = 1.
// Gradient operands are scaled by the power-of-two loss scale S (see dib_enc_fused.cu) to stay inside fp16 range.
//
// The GEMM kernels are warp-specialised: warps 0..7 are two consumer warpgroups (warpgroup g computes rows [64 g, 64 g + 64)
// of the 128-row tile with m64nNk16 wgmma instructions, accumulators in registers, and runs the epilogue), warp 8 issues
// the TMA loads of the shared-memory ring.
#include <cuda.h>
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <stdlib.h>

#include "dib_common.cuh"
#include "dib_kernels.h"
#include "dib_sm90.cuh"

int dib_int16_rb_enabled();
int dib_int16_head1_enabled();

namespace {

using namespace sm90;

constexpr int kBM = 128, kBN = 128, kBK = 64, kStages = 3, kRbStages = 4;
constexpr int kABytes = kBM * 128, kBBytes = kBN * 128, kStageBytes = kABytes + kBBytes;
constexpr int kConsumers = 256, kGemmThreads = kConsumers + 32;
constexpr int kProducerWarp = kConsumers / 32;
constexpr int kEmptyArrivals = kConsumers / 32;   // every consumer warp releases a stage once its MMAs have read it

struct Int16Args {
  float* out32; uint16_t* out16; int ldc;       // WGRAD partial base (fp32) | FWD/DGRAD output (fp16)
  const uint16_t* X; int ldx;                   // DGRAD: activation whose act' gates the gradient (or null)
  const float* bias;                          // FWD
  float* dbias;                               // DGRAD: column sums of the produced gradient per 128-row tile [tiles_r][C] (or null)
  int M, T, C, R, act;
  float alpha, out_scale;
  int nsplit, rows_per_split; long long split_stride;
  int dbg;                                    // measurement only (dib_debug_set_variant key 5): 1 = skip the epilogue's global stores
};

template <bool BF16>
__device__ __forceinline__ uint32_t pack_h2(float a, float b) {
  uint32_t r;
  if constexpr (BF16) asm("cvt.rn.satfinite.bf16x2.f32 %0, %1, %2;" : "=r"(r) : "f"(b), "f"(a));
  else asm("cvt.rn.satfinite.f16x2.f32 %0, %1, %2;" : "=r"(r) : "f"(b), "f"(a));
  return r;
}
template <bool BF16>
__device__ __forceinline__ void unpack_h2(uint32_t u, float& a, float& b) {
  if constexpr (BF16) { a = __uint_as_float(u << 16); b = __uint_as_float(u & 0xffff0000u); }
  else { const float2 f = __half22float2(*reinterpret_cast<__half2*>(&u)); a = f.x; b = f.y; }
}

__device__ __forceinline__ void st_shared_b32(uint32_t addr, uint32_t v) {
  asm volatile("st.shared.b32 [%0], %1;" ::"r"(addr), "r"(v) : "memory");
}

// 16-bit operand tiles of one pipeline stage (TMA SWIZZLE_128B boxes, see map_k / map_mn):
//   K-major  [rows][128 B]: a 16-deep k step is 32 B;  warpgroup g's 64 rows start 8 KB in
//   MN-major [panels of 64 M/N][64 k-rows][128 B]: a 16-deep k step is 2048 B, panels 8 KB apart
__device__ __forceinline__ uint64_t desc_kmaj(uint32_t base, int kk) { return gmma_desc(base + kk * 32, 16, 1024); }
__device__ __forceinline__ uint64_t desc_mnmaj(uint32_t base, int kk) { return gmma_desc(base + kk * 2048, kBK * 128, 1024); }

// the 8 lanes of a warp that share lane % 4 hold the same accumulator columns: sum them (fixed order); lanes 0..3 get the total
__device__ __forceinline__ float quad_col_sum(float v) {
  v += __shfl_xor_sync(0xffffffffu, v, 4);
  v += __shfl_xor_sync(0xffffffffu, v, 8);
  v += __shfl_xor_sync(0xffffffffu, v, 16);
  return v;
}

// Persistent: each CTA walks tiles blockIdx.x, +gridDim.x, ...; the shared-memory stage ring runs across tiles, and two
// CTAs per SM let one CTA's epilogue overlap the other's mainloop.
// RB (FWD / DGRAD only): "resident B" -- each CTA owns ONE column tile, loads its [K x 128] slice of the weights once and
// streams only the activation tiles; the MMAs and the epilogue are those of the streamed variant, so the results are
// bit-identical.
template <int MODE, bool BF16, bool RB>
__global__ void __launch_bounds__(kGemmThreads, RB ? 1 : 2)
dib_int16_gemm_kernel(const __grid_constant__ CUtensorMap mapA, const __grid_constant__ CUtensorMap mapB, const Int16Args a,
                      const __grid_constant__ CUtensorMap mapA2, const __grid_constant__ CUtensorMap mapB2, const Int16Args a2, int nkb) {
  // (a2, mapA2, mapB2): an optional SECOND weight-gradient problem walked by the same launch (a2.nsplit > 0, WGRAD only): the two
  // layers' tiles together fill one wave of CTAs, which neither fills alone
  static_assert(!RB || MODE != DIB_GEMM_WGRAD, "resident-B variant: FWD / DGRAD only");
  constexpr bool A_MN = (MODE == DIB_GEMM_WGRAD), B_MN = (MODE != DIB_GEMM_DGRAD);
  constexpr int S = RB ? kRbStages : kStages;
  constexpr uint32_t kStep = RB ? kABytes : kStageBytes;          // bytes per ring stage
  extern __shared__ uint8_t smem_raw[];
  const uint32_t sb = (smem_u32(smem_raw) + 1023u) & ~1023u;
  const uint32_t sBres = sb, ring = RB ? sb + nkb * kBBytes : sb;  // RB: resident weight slice, then the A ring
  const uint32_t bar_base = ring + S * kStep;
  auto full_bar = [&](int s) { return bar_base + 8u * s; };
  auto empty_bar = [&](int s) { return bar_base + 8u * (S + s); };
  const uint32_t bfull_bar = bar_base + 8u * (2 * S);

  __shared__ float colsum_s[kConsumers / 32][kBN];
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int R0 = (MODE == DIB_GEMM_WGRAD) ? a.R : a.M, C0 = a.C;
  const int tiles_r = DIB_CEIL_DIV(R0, kBM), tiles_c = DIB_CEIL_DIV(C0, kBN);
  const int nsp = (MODE == DIB_GEMM_WGRAD) ? a.nsplit : 1;
  const int ntile0 = tiles_r * tiles_c * nsp;
  const bool two = (MODE == DIB_GEMM_WGRAD) && a2.nsplit > 0;
  const int tiles_r2 = two ? DIB_CEIL_DIV(a2.R, kBM) : 0, tiles_c2 = two ? DIB_CEIL_DIV(a2.C, kBN) : 0;
  const int ntile = RB ? tiles_r : ntile0 + tiles_r2 * tiles_c2 * (two ? a2.nsplit : 0);
  // RB: this CTA's fixed column tile and its row tiles: blockIdx.x = col + tiles_c * k  (gridDim.x is a multiple of tiles_c)
  const int rb_c0 = RB ? (blockIdx.x % tiles_c) * kBN : 0;
  const int first = RB ? blockIdx.x / tiles_c : blockIdx.x, stride = RB ? gridDim.x / tiles_c : gridDim.x;

  int prob = 0;                                     // which problem the tile last decoded belongs to (per thread)
  auto decode = [&](int tile, int& r0, int& c0, int& split, int& t_begin, int& nk) {
    if (RB) { prob = 0; split = 0; r0 = tile * kBM; c0 = rb_c0; t_begin = 0; nk = nkb; return; }
    prob = (two && tile >= ntile0) ? 1 : 0;
    if (prob) tile -= ntile0;
    const int tr = prob ? tiles_r2 : tiles_r, tcn = prob ? tiles_c2 : tiles_c;
    const int per = tr * tcn;
    split = tile / per;
    const int rem = tile - split * per;
    r0 = (rem / tcn) * kBM; c0 = (rem % tcn) * kBN;
    int t_end;
    if (MODE == DIB_GEMM_WGRAD) {
      const int rps = prob ? a2.rows_per_split : a.rows_per_split;
      t_begin = split * rps; t_end = min(a.M, t_begin + rps);
    } else { t_begin = 0; t_end = a.T; }
    nk = t_end > t_begin ? DIB_CEIL_DIV(t_end - t_begin, kBK) : 0;
  };

  if (tid == 0) {
    for (int s = 0; s < S; ++s) { mbar_init(full_bar(s), 1); mbar_init(empty_bar(s), kEmptyArrivals); }
    mbar_init(bfull_bar, 1);
    fence_barrier_init();
  }
  __syncthreads();

  if (warp == kProducerWarp) {
    // ============================================================== TMA producer (one lane)
    if (lane == 0) {
      tma_prefetch_desc(&mapA); tma_prefetch_desc(&mapB);
      if (two) { tma_prefetch_desc(&mapA2); tma_prefetch_desc(&mapB2); }
      if constexpr (RB) {                           // the weight slice of this column tile, once
        mbar_expect_tx(bfull_bar, (uint32_t)(nkb * kBBytes));
        for (int k = 0; k < nkb; ++k) {
          // one box per k-block: FWD [2 panels][64 k-rows][128 B] (MN-major), DGRAD [128 rows][128 B] (K-major)
          if constexpr (B_MN) tma_load_3d(sBres + k * kBBytes, &mapB, bfull_bar, 0, k * kBK, rb_c0 / 64);
          else                tma_load_2d(sBres + k * kBBytes, &mapB, bfull_bar, k * kBK, rb_c0);
        }
      }
      uint32_t s = 0, ph = 0;
      for (int tile = first; tile < ntile; tile += stride) {
        int r0, c0, split, t_begin, nk;
        decode(tile, r0, c0, split, t_begin, nk);
        const CUtensorMap* mA = prob ? &mapA2 : &mapA;
        const CUtensorMap* mB = prob ? &mapB2 : &mapB;
        for (int k = 0; k < nk; ++k) {
          mbar_wait(empty_bar(s), ph ^ 1);
          mbar_expect_tx(full_bar(s), kStep);
          const uint32_t a_dst = ring + s * kStep, b_dst = a_dst + kABytes;
          const int t0 = t_begin + k * kBK;
          if constexpr (A_MN) tma_load_3d(a_dst, mA, full_bar(s), 0, t0, r0 / 64);
          else                tma_load_2d(a_dst, mA, full_bar(s), t0, r0);
          if constexpr (!RB) {
            if constexpr (B_MN) tma_load_3d(b_dst, mB, full_bar(s), 0, t0, c0 / 64);
            else                tma_load_2d(b_dst, mB, full_bar(s), t0, c0);
          }
          if (++s == S) { s = 0; ph ^= 1; }
        }
      }
    }
  } else {
    // ============================================================== consumer warpgroups: MMAs + epilogue
    const int wg = tid >> 7, q = lane & 3;
    const int rb = 64 * wg + 16 * (warp & 3) + (lane >> 2);       // tile row of this thread's accumulator elements
    if constexpr (RB) mbar_wait(bfull_bar, 0);
    uint32_t s = 0, ph = 0;
    for (int tile = first; tile < ntile; tile += stride) {
      int r0, c0, split, t_begin, nk;
      decode(tile, r0, c0, split, t_begin, nk);
      float acc[64];
#pragma unroll
      for (int i = 0; i < 64; ++i) acc[i] = 0.f;
      if (nk > 0) {
        uint32_t prev = 0;
        for (int k = 0; k < nk; ++k) {
          mbar_wait(full_bar(s), ph);
          const uint32_t a_base = ring + s * kStep;
          const uint32_t b_base = RB ? sBres + k * kBBytes : a_base + kABytes;
          wgmma_fence();
#pragma unroll
          for (int kk = 0; kk < kBK / 16; ++kk) {
            const uint64_t da = A_MN ? desc_mnmaj(a_base + wg * (kBK * 128), kk) : desc_kmaj(a_base + wg * 64 * 128, kk);
            const uint64_t db = B_MN ? desc_mnmaj(b_base, kk) : desc_kmaj(b_base, kk);
            wgmma_m64n128k16<BF16, A_MN ? 1 : 0, B_MN ? 1 : 0>(acc, da, db, (k > 0 || kk > 0) ? 1u : 0u);
          }
          wgmma_commit();
          wgmma_wait<1>();                                        // the previous stage's MMAs have read their operands
          if (k > 0 && lane == 0) mbar_arrive(empty_bar(prev));
          prev = s;
          if (++s == S) { s = 0; ph ^= 1; }
        }
        wgmma_wait<0>();
        if (lane == 0) mbar_arrive(empty_bar(prev));
        wgmma_fence_regs(acc);
      }
      // ---------------- epilogue: rows r0 + rb (+8), columns c0 + 8 j + 2 q (+1)
      const int R = prob ? a2.R : R0, C = prob ? a2.C : C0;
      float* const out32 = prob ? a2.out32 : a.out32;
      const int ldc32 = prob ? a2.ldc : a.ldc;
#pragma unroll
      for (int j = 0; j < kBN / 8; ++j) {
        const int c = c0 + 8 * j + 2 * q;
        const bool cl = c < C;                              // C is even: a column pair is entirely inside or outside
        float cs[2] = {0.f, 0.f};
        float2 bias = make_float2(0.f, 0.f);
        if constexpr (MODE == DIB_GEMM_FWD) { if (cl) bias = *reinterpret_cast<const float2*>(a.bias + c); }
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          const int r = r0 + rb + 8 * h;
          const bool live = cl && r < R;
          float v0 = acc[4 * j + 2 * h], v1 = acc[4 * j + 2 * h + 1];
          if constexpr (MODE == DIB_GEMM_WGRAD) {
            if (live && !(a.dbg & 1))
              *reinterpret_cast<float2*>(out32 + (long long)split * a.split_stride + (long long)r * ldc32 + c) =
                  make_float2(v0 * a.out_scale, v1 * a.out_scale);
          } else {
            if constexpr (MODE == DIB_GEMM_FWD) {
              v0 = dib_act16(a.act, v0 + bias.x, a.alpha);
              v1 = dib_act16(a.act, v1 + bias.y, a.alpha);
            } else if (a.X) {
              float x0 = 0.f, x1 = 0.f;
              if (live) unpack_h2<BF16>(*reinterpret_cast<const uint32_t*>(a.X + (long long)r * a.ldx + c), x0, x1);
              v0 *= dib_act_grad(a.act, x0, a.alpha);
              v1 *= dib_act_grad(a.act, x1, a.alpha);
            }
            if (live && !(a.dbg & 1)) *reinterpret_cast<uint32_t*>(a.out16 + (long long)r * a.ldc + c) = pack_h2<BF16>(v0, v1);
            if (live) { cs[0] += v0; cs[1] += v1; }               // rows / columns outside the matrix add nothing
          }
        }
        if constexpr (MODE == DIB_GEMM_DGRAD) {
          if (a.dbias) {
            // bias gradient of the layer below = column sums of the gradient just produced: the warp's 16 rows here, the 8
            // warps of the tile below
            cs[0] = quad_col_sum(cs[0]); cs[1] = quad_col_sum(cs[1]);
            if (lane < 4) { colsum_s[warp][8 * j + 2 * q] = cs[0]; colsum_s[warp][8 * j + 2 * q + 1] = cs[1]; }
          }
        }
      }
      if constexpr (MODE == DIB_GEMM_DGRAD) {
        if (a.dbias) {
          named_bar_sync(1, kConsumers);
          if (tid < kBN && c0 + tid < C) {
            float sum = 0.f;
#pragma unroll
            for (int w = 0; w < kConsumers / 32; ++w) sum += colsum_s[w][tid];
            a.dbias[(long long)(r0 / kBM) * C + c0 + tid] = sum;
          }
          named_bar_sync(1, kConsumers);
        }
      }
    }
  }
}

// ====================================================================================================
// Fused tail of the integration network for single-output models (C0, nb-radial): the last two hidden layers
// (256 wide each) and the output head in ONE persistent kernel -- models.py:81-84,122 + the compiled loss.
//   per 128-row tile:  L0  D0 = A W0   (A, W0 k-blocks streamed through a TMA ring; N = 256, fp32 in registers)
//                      e0  g1 = act(D0 + b0) -> 16-bit -> swizzled shared tile (= L1's A operand) and -> HBM (the backward needs it)
//                      L1  D1 = g1 W1  (W1 k-blocks through the same ring)
//                      e1  g2 = act(D1 + b1) kept PACKED IN REGISTERS, logit = g2 . w + b, compiled loss / metric,
//                          d loss / d logit, dg2 = dz w act'(g2) -> HBM, output-layer weight / bias gradients and the bias gradient
//                          of the last hidden layer as per-CTA partials.
// g2 never reaches HBM, and the head's re-read of it (and its launch) disappears.  A warp owns 16 whole rows of the
// accumulator, so each row's logit is complete after a reduction over the 4 lanes that share the row.
// ====================================================================================================
constexpr int kF2N = 256, kF2Stages = 2;
constexpr int kF2AB = kBM * 128, kF2BB = kF2N * 128, kF2Stage = kF2AB + kF2BB;      // 16 KB + 32 KB
constexpr int kF2G1Off = kF2Stages * kF2Stage;
constexpr int kF2BarOff = kF2G1Off + kBM * kF2N * 2;
constexpr int kF2Smem = kF2BarOff + 64 + 1024;

struct Fwd2Args {
  const float *b0, *b1, *wout, *bout;
  uint16_t* g1; int ldg1;             // out: first fused layer's activation [M x 256]
  uint16_t* dg2; int lddg;            // out (training) or null: gradient w.r.t. the second fused layer's pre-activation, x gscale
  const float* y; float* user_pred;
  float* wpart; int wpart_stride; float *loss_part, *acc_part;
  int M, nk0, act, out_act, loss;
  float alpha, inv_batch, gscale;
};

// ACT is a template parameter: the activation switch inside the fully unrolled register-resident passes would otherwise be
// evaluated per element.
constexpr int kF2Threads = kConsumers + 128;      // + a producer warpgroup, so that setmaxnreg can move its registers to the consumers
template <bool BF16, int ACT>
__global__ void __launch_bounds__(kF2Threads, 1)
dib_int16_fwd2_kernel(const __grid_constant__ CUtensorMap mapA, const __grid_constant__ CUtensorMap mapW0,
                      const __grid_constant__ CUtensorMap mapW1, const Fwd2Args a) {
  extern __shared__ uint8_t smem_raw[];
  const uint32_t sb = (smem_u32(smem_raw) + 1023u) & ~1023u;
  const uint32_t bar_base = sb + kF2BarOff;
  auto full_bar = [&](int s) { return bar_base + 8u * s; };
  auto empty_bar = [&](int s) { return bar_base + 8u * (kF2Stages + s); };
  const uint32_t g1s = sb + kF2G1Off;

  __shared__ __align__(16) float s_b0[kF2N], s_b1[kF2N], s_w[kF2N];
  __shared__ float s_colw[kConsumers / 32][kF2N], s_colb[kConsumers / 32][kF2N];
  __shared__ float s_red[3][kConsumers / 32];
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int ntile = DIB_CEIL_DIV(a.M, kBM);

  for (int i = tid; i < kF2N; i += blockDim.x) { s_b0[i] = a.b0[i]; s_b1[i] = a.b1[i]; s_w[i] = a.wout[i]; }
  if (tid == 0) {
    for (int s = 0; s < kF2Stages; ++s) { mbar_init(full_bar(s), 1); mbar_init(empty_bar(s), kEmptyArrivals); }
    fence_barrier_init();
  }
  __syncthreads();

  if (warp >= kProducerWarp) {
    asm volatile("setmaxnreg.dec.sync.aligned.u32 40;");
    if (warp == kProducerWarp && lane == 0) {
      tma_prefetch_desc(&mapA); tma_prefetch_desc(&mapW0); tma_prefetch_desc(&mapW1);
      uint32_t s = 0, ph = 0;
      for (int tile = blockIdx.x; tile < ntile; tile += gridDim.x) {
        for (int k = 0; k < a.nk0; ++k) {
          mbar_wait(empty_bar(s), ph ^ 1);
          mbar_expect_tx(full_bar(s), kF2Stage);
          const uint32_t dst = sb + s * kF2Stage;
          tma_load_2d(dst, &mapA, full_bar(s), k * kBK, tile * kBM);
          tma_load_3d(dst + kF2AB, &mapW0, full_bar(s), 0, k * kBK, 0);
          if (++s == kF2Stages) { s = 0; ph ^= 1; }
        }
        for (int k = 0; k < kF2N / kBK; ++k) {
          mbar_wait(empty_bar(s), ph ^ 1);
          mbar_expect_tx(full_bar(s), kF2BB);
          tma_load_3d(sb + s * kF2Stage + kF2AB, &mapW1, full_bar(s), 0, k * kBK, 0);
          if (++s == kF2Stages) { s = 0; ph ^= 1; }
        }
      }
    }
    return;
  }
  asm volatile("setmaxnreg.inc.sync.aligned.u32 232;");   // 128 x 40 + 256 x 232 <= 64 K registers

  const int wg = tid >> 7, q = lane & 3;
  const int rb = 64 * wg + 16 * (warp & 3) + (lane >> 2);
  const bool train = a.dg2 != nullptr;
  const float bout = a.bout[0];
  float acc_dw = 0.f, acc_dbh = 0.f, lsum = 0.f, asum = 0.f, dbo = 0.f;     // column accumulators: column tid
  uint32_t s = 0, ph = 0;
  // one k-loop of m64n256k16 MMAs over `nk` ring stages; A from the ring (a_ring) or the shared g1 tile
  auto mainloop = [&](float (&acc)[128], int nk, bool a_ring) {
    uint32_t prev = 0;
    for (int k = 0; k < nk; ++k) {
      mbar_wait(full_bar(s), ph);
      const uint32_t st = sb + s * kF2Stage;
      const uint32_t a_base = a_ring ? st + wg * 64 * 128 : g1s + k * kF2AB + wg * 64 * 128;
      wgmma_fence();
#pragma unroll
      for (int kk = 0; kk < kBK / 16; ++kk)
        wgmma_m64n256k16<BF16, 0, 1>(acc, desc_kmaj(a_base, kk), desc_mnmaj(st + kF2AB, kk), (k > 0 || kk > 0) ? 1u : 0u);
      wgmma_commit();
      wgmma_wait<1>();
      if (k > 0 && lane == 0) mbar_arrive(empty_bar(prev));
      prev = s;
      if (++s == kF2Stages) { s = 0; ph ^= 1; }
    }
    wgmma_wait<0>();
    if (lane == 0) mbar_arrive(empty_bar(prev));
    wgmma_fence_regs(acc);
  };

  for (int tile = blockIdx.x; tile < ntile; tile += gridDim.x) {
    const long long row_lo = (long long)tile * kBM + rb;
    float acc[128];
#pragma unroll
    for (int i = 0; i < 128; ++i) acc[i] = 0.f;
    // ---------------- L0, e0: g1 = act(D0 + b0) -> shared tile (L1's A operand) and HBM
    mainloop(acc, a.nk0, true);
#pragma unroll
    for (int j = 0; j < kF2N / 8; ++j) {
      const int c = 8 * j + 2 * q;
      const float2 bv = *reinterpret_cast<const float2*>(&s_b0[c]);
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int r = rb + 8 * h;
        const uint32_t w = pack_h2<BF16>(dib_act16(ACT, acc[4 * j + 2 * h] + bv.x, a.alpha), dib_act16(ACT, acc[4 * j + 2 * h + 1] + bv.y, a.alpha));
        st_shared_b32(g1s + (c >> 6) * kF2AB + r * 128 + ((((c & 63) >> 3) ^ (r & 7)) << 4) + 4 * q, w);
        if (row_lo + 8 * h < a.M) *reinterpret_cast<uint32_t*>(a.g1 + (row_lo + 8 * h) * a.ldg1 + c) = w;
      }
    }
    fence_proxy_async_smem();
    named_bar_sync(2 + wg, 128);                     // this warpgroup's rows of g1 are complete
    // ---------------- L1, e1 pass 1: g2 = act(D1 + b1) packed into registers, partial logits
#pragma unroll
    for (int i = 0; i < 128; ++i) acc[i] = 0.f;
    mainloop(acc, kF2N / kBK, false);
    uint32_t g2p[64];
    float zp[2] = {0.f, 0.f};
#pragma unroll
    for (int j = 0; j < kF2N / 8; ++j) {
      const int c = 8 * j + 2 * q;
      const float2 bv = *reinterpret_cast<const float2*>(&s_b1[c]), wv = *reinterpret_cast<const float2*>(&s_w[c]);
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const uint32_t p = pack_h2<BF16>(dib_act16(ACT, acc[4 * j + 2 * h] + bv.x, a.alpha), dib_act16(ACT, acc[4 * j + 2 * h + 1] + bv.y, a.alpha));
        g2p[2 * j + h] = p;
        float h0, h1;
        unpack_h2<BF16>(p, h0, h1);
        zp[h] = fmaf(h0, wv.x, zp[h]); zp[h] = fmaf(h1, wv.y, zp[h]);
      }
    }
    // ---------------- logit, compiled loss / metric, d loss / d logit (the 4 lanes of a row compute it; lane q = 0 accumulates)
    float dzs[2], ds[2];
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      zp[h] += __shfl_xor_sync(0xffffffffu, zp[h], 1);
      zp[h] += __shfl_xor_sync(0xffffffffu, zp[h], 2);
      const long long row = row_lo + 8 * h;
      const bool live = row < a.M;
      const float z = dib_act(a.out_act, zp[h] + bout, a.alpha);
      float dz = 0.f;
      if (live && a.y) {
        const float t = a.y[row];
        float l;
        if (a.loss == DIB_LOSS_BCE_LOGITS) { l = fmaxf(z, 0.f) - z * t + log1pf(expf(-fabsf(z))); dz = 1.f / (1.f + expf(-z)) - t; }
        else if (a.loss == DIB_LOSS_BCE_PROBS) {
          const float ep = 1e-7f, pc = fminf(fmaxf(z, ep), 1.f - ep);
          l = -(t * logf(pc + ep) + (1.f - t) * logf(1.f - pc + ep));
          dz = (z > ep && z < 1.f - ep) ? -t / (pc + ep) + (1.f - t) / (1.f - pc + ep) : 0.f;
        } else if (a.loss == DIB_LOSS_SPARSE_CE_LOGITS) { l = 0.f; dz = 0.f; }        // one class: the softmax is constant
        else { const float d = z - t; l = d * d; dz = 2.f * d; }
        const float acc1 = a.loss == DIB_LOSS_SPARSE_CE_LOGITS ? ((int)t == 0 ? 1.f : 0.f) : (((z > 0.5f ? 1.f : 0.f) == t) ? 1.f : 0.f);
        if (q == 0) { lsum += l; asum += acc1; }
      }
      if (a.user_pred && live && q == 0) a.user_pred[row] = z;
      dzs[h] = live ? dz * a.inv_batch * dib_act_grad(a.out_act, z, a.alpha) : 0.f;
      ds[h] = dzs[h] * a.gscale;
      if (q == 0) dbo += dzs[h];
    }
    if (train) {
      // ---------------- e1, pass 2: dg2 = ds w act'(g2) -> HBM; column sums of g2 dz (output-layer dW) and of dg2 (bias gradient)
#pragma unroll
      for (int j = 0; j < kF2N / 8; ++j) {
        const int c = 8 * j + 2 * q;
        const float2 wv = *reinterpret_cast<const float2*>(&s_w[c]);
        float cw[2] = {0.f, 0.f}, cb[2] = {0.f, 0.f};
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          float h0, h1;
          unpack_h2<BF16>(g2p[2 * j + h], h0, h1);
          const float d0 = ds[h] * wv.x * dib_act_grad(ACT, h0, a.alpha), d1 = ds[h] * wv.y * dib_act_grad(ACT, h1, a.alpha);
          cw[0] += h0 * dzs[h]; cw[1] += h1 * dzs[h];
          cb[0] += d0; cb[1] += d1;
          if (row_lo + 8 * h < a.M) *reinterpret_cast<uint32_t*>(a.dg2 + (row_lo + 8 * h) * a.lddg + c) = pack_h2<BF16>(d0, d1);
        }
#pragma unroll
        for (int k = 0; k < 2; ++k) {
          cw[k] = quad_col_sum(cw[k]);
          cb[k] = quad_col_sum(cb[k]);
        }
        if (lane < 4) {
          s_colw[warp][c] = cw[0]; s_colw[warp][c + 1] = cw[1];
          s_colb[warp][c] = cb[0]; s_colb[warp][c + 1] = cb[1];
        }
      }
      // the 8 warps cover the tile's 128 rows: fixed-order combine into the thread-owned column
      named_bar_sync(1, kConsumers);
#pragma unroll
      for (int w = 0; w < kConsumers / 32; ++w) { acc_dw += s_colw[w][tid]; acc_dbh += s_colb[w][tid]; }
      named_bar_sync(1, kConsumers);
    }
  }
  // ---------------- per-CTA partials, layout of the head kernels: [dWc (K) | dbc (1) | column sums of dg2 (K)], loss, accuracy
  if (train) {
    a.wpart[(long long)blockIdx.x * a.wpart_stride + tid] = acc_dw;
    a.wpart[(long long)blockIdx.x * a.wpart_stride + kF2N + 1 + tid] = acc_dbh;
  }
  lsum = dib_warp_sum(lsum); asum = dib_warp_sum(asum); dbo = dib_warp_sum(dbo);
  if (lane == 0) { s_red[0][warp] = lsum; s_red[1][warp] = asum; s_red[2][warp] = dbo; }
  named_bar_sync(1, kConsumers);
  if (tid == 0) {
    float l = 0.f, ac = 0.f, b = 0.f;
    for (int w = 0; w < kConsumers / 32; ++w) { l += s_red[0][w]; ac += s_red[1][w]; b += s_red[2][w]; }
    a.loss_part[blockIdx.x] = l;
    a.acc_part[blockIdx.x] = ac;
    if (train) a.wpart[(long long)blockIdx.x * a.wpart_stride + kF2N] = b;
  }
}

// ----------------------------------------------------------------------------------------------------
// output head: one warp per row; lanes own 8 hidden units each (K = 256) or loop (K = multiple of 256)
// ----------------------------------------------------------------------------------------------------
constexpr int kHeadMaxOut = 16, kHeadWarps = 8;

template <int KPT, int OUT, int ROWS, bool BF16>   // hidden units per lane (K / 32); bound of the output width; rows in flight per warp
__global__ void __launch_bounds__(kHeadWarps * 32)
dib_int16_head_kernel(const uint16_t* __restrict__ g, int ldg, int K, const float* __restrict__ Wc, const float* __restrict__ bc,
                      int out_dim, int out_act, int hid_act, float alpha, int loss, const float* __restrict__ y, long long n,
                      float inv_batch, float gscale, uint16_t* __restrict__ dg, int lddg, float* __restrict__ user_pred,
                      float* __restrict__ wpart, int wpart_stride, float* __restrict__ loss_part, float* __restrict__ acc_part) {
  __shared__ float red[kHeadWarps][KPT * 32];
  __shared__ float sred[kHeadWarps];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int gw = blockIdx.x * kHeadWarps + warp, nw = gridDim.x * kHeadWarps;
  float w[KPT][OUT], dw[KPT][OUT], db[OUT], bias[OUT], dbh[KPT];
#pragma unroll
  for (int i = 0; i < KPT; ++i) dbh[i] = 0.f;
#pragma unroll
  for (int o = 0; o < OUT; ++o) {
    db[o] = 0.f;
    bias[o] = o < out_dim ? bc[o] : 0.f;
#pragma unroll
    for (int i = 0; i < KPT; ++i) {
      w[i][o] = o < out_dim ? Wc[(long long)(lane * KPT + i) * out_dim + o] : 0.f;
      dw[i][o] = 0.f;
    }
  }
  float lsum = 0.f, asum = 0.f;
  const bool train = dg != nullptr;

  for (long long row0 = (long long)gw * ROWS; row0 < n; row0 += (long long)nw * ROWS) {
    uint4 hv[ROWS][KPT / 8];
#pragma unroll
    for (int rr = 0; rr < ROWS; ++rr) {                 // issue all loads of the row group first (memory-level parallelism)
      const long long row = row0 + rr < n ? row0 + rr : n - 1;
#pragma unroll
      for (int i = 0; i < KPT; i += 8) hv[rr][i / 8] = *reinterpret_cast<const uint4*>(g + row * ldg + lane * KPT + i);
    }
#pragma unroll
    for (int rr = 0; rr < ROWS; ++rr) {
      const long long row = row0 + rr;
      if (row >= n) break;
      float h[KPT];
#pragma unroll
      for (int i = 0; i < KPT; i += 8) {
        const uint4 v = hv[rr][i / 8];
        unpack_h2<BF16>(v.x, h[i], h[i + 1]); unpack_h2<BF16>(v.y, h[i + 2], h[i + 3]);
        unpack_h2<BF16>(v.z, h[i + 4], h[i + 5]); unpack_h2<BF16>(v.w, h[i + 6], h[i + 7]);
      }
      float z[OUT], dz[OUT];
#pragma unroll
      for (int o = 0; o < OUT; ++o) {
        float s = 0.f;
#pragma unroll
        for (int i = 0; i < KPT; ++i) s = fmaf(h[i], w[i][o], s);
        z[o] = dib_act(out_act, dib_warp_sum(s) + bias[o], alpha);
        dz[o] = 0.f;
      }
      // ---- compiled loss / metric / d loss / d z  (identical on all lanes)
      if (y) {
        float l = 0.f, acc = 0.f;
        const float inv_out = 1.f / (float)out_dim;
        if (loss == DIB_LOSS_SPARSE_CE_LOGITS) {
          const int label = (int)y[row];
          float m = z[0], zl = 0.f, se = 0.f; int am = 0;
#pragma unroll
          for (int o = 1; o < OUT; ++o) if (o < out_dim && z[o] > m) { m = z[o]; am = o; }
#pragma unroll
          for (int o = 0; o < OUT; ++o) if (o < out_dim) { se += expf(z[o] - m); if (o == label) zl = z[o]; }
          l = m + logf(se) - zl;
          acc = am == label ? 1.f : 0.f;
#pragma unroll
          for (int o = 0; o < OUT; ++o) if (o < out_dim) dz[o] = expf(z[o] - m) / se - (o == label ? 1.f : 0.f);
        } else {
#pragma unroll
          for (int o = 0; o < OUT; ++o) if (o < out_dim) {
            const float t = y[row * out_dim + o];
            if (loss == DIB_LOSS_BCE_LOGITS) { l += fmaxf(z[o], 0.f) - z[o] * t + log1pf(expf(-fabsf(z[o]))); dz[o] = (1.f / (1.f + expf(-z[o])) - t) * inv_out; }
            else if (loss == DIB_LOSS_BCE_PROBS) {
              const float ep = 1e-7f, pc = fminf(fmaxf(z[o], ep), 1.f - ep);
              l -= t * logf(pc + ep) + (1.f - t) * logf(1.f - pc + ep);
              dz[o] = (z[o] > ep && z[o] < 1.f - ep) ? (-t / (pc + ep) + (1.f - t) / (1.f - pc + ep)) * inv_out : 0.f;
            } else { const float d = z[o] - t; l += d * d; dz[o] = 2.f * d * inv_out; }
            acc += ((z[o] > 0.5f ? 1.f : 0.f) == t) ? 1.f : 0.f;
          }
          l *= inv_out; acc *= inv_out;
        }
        lsum += l; asum += acc;
      }
      if (user_pred) {
#pragma unroll
        for (int o = 0; o < OUT; ++o) if (o < out_dim && lane == o) user_pred[row * out_dim + o] = z[o];
      }
      if (train) {
#pragma unroll
        for (int o = 0; o < OUT; ++o) { dz[o] *= inv_batch * dib_act_grad(out_act, z[o], alpha); db[o] += dz[o]; }
        float d[KPT];
#pragma unroll
        for (int i = 0; i < KPT; ++i) {
          float s = 0.f;
#pragma unroll
          for (int o = 0; o < OUT; ++o) { s = fmaf(dz[o], w[i][o], s); dw[i][o] = fmaf(h[i], dz[o], dw[i][o]); }
          d[i] = s * gscale * dib_act_grad(hid_act, h[i], alpha);
          dbh[i] += d[i];
        }
        uint16_t* dst = dg + row * lddg + lane * KPT;
#pragma unroll
        for (int i = 0; i < KPT; i += 8)
          *reinterpret_cast<uint4*>(dst + i) = make_uint4(pack_h2<BF16>(d[i], d[i + 1]), pack_h2<BF16>(d[i + 2], d[i + 3]),
                                                          pack_h2<BF16>(d[i + 4], d[i + 5]), pack_h2<BF16>(d[i + 6], d[i + 7]));
      }
    }
  }
  // ---- per-block partials (fixed order over the block's warps): output-layer weight/bias gradients, loss, accuracy
  if (train) {
#pragma unroll
    for (int o = 0; o < OUT; ++o) {
      if (o < out_dim) {
#pragma unroll
        for (int i = 0; i < KPT; ++i) red[warp][lane * KPT + i] = dw[i][o];
      }
      __syncthreads();
      if (warp == 0 && o < out_dim) {
#pragma unroll
        for (int i = 0; i < KPT; ++i) {
          float s = 0.f;
          for (int ww = 0; ww < kHeadWarps; ++ww) s += red[ww][lane * KPT + i];
          wpart[(long long)blockIdx.x * wpart_stride + (long long)(lane * KPT + i) * out_dim + o] = s;
        }
      }
      __syncthreads();
    }
    // bias gradient of the last hidden layer (column sums of dg, still multiplied by gscale) -> wpart[K*out+out + k]
#pragma unroll
    for (int i = 0; i < KPT; ++i) red[warp][lane * KPT + i] = dbh[i];
    __syncthreads();
    if (warp == 0) {
#pragma unroll
      for (int i = 0; i < KPT; ++i) {
        float s = 0.f;
        for (int ww = 0; ww < kHeadWarps; ++ww) s += red[ww][lane * KPT + i];
        wpart[(long long)blockIdx.x * wpart_stride + (long long)K * out_dim + out_dim + lane * KPT + i] = s;
      }
    }
    __syncthreads();
    if (lane == 0) {
#pragma unroll
      for (int o = 0; o < OUT; ++o) red[warp][o] = db[o];
    }
    __syncthreads();
    if (threadIdx.x < out_dim) {
      float s = 0.f;
      for (int ww = 0; ww < kHeadWarps; ++ww) s += red[ww][threadIdx.x];
      wpart[(long long)blockIdx.x * wpart_stride + (long long)K * out_dim + threadIdx.x] = s;
    }
    __syncthreads();
  }
  if (lane == 0) sred[warp] = lsum;
  __syncthreads();
  if (threadIdx.x == 0) { float s = 0.f; for (int ww = 0; ww < kHeadWarps; ++ww) s += sred[ww]; loss_part[blockIdx.x] = s; }
  __syncthreads();
  if (lane == 0) sred[warp] = asum;
  __syncthreads();
  if (threadIdx.x == 0) { float s = 0.f; for (int ww = 0; ww < kHeadWarps; ++ww) s += sred[ww]; acc_part[blockIdx.x] = s; }
}


// ----------------------------------------------------------------------------------------------------
// output head, single-output specialisation (C0, nb-radial: out = 1).  Same mapping as above (a warp per row, 8 hidden
// units per lane) but 8 rows per pass: the eight row dot products are reduced with ONE transposing butterfly (9 shuffles
// instead of 40), after which lane L holds the logit of row L & 7 and the loss / metric / d loss / d z arithmetic runs once
// per pass, lane-parallel, instead of once per row on every lane (ncu: the generic kernel was issue-bound at 45 %).
// ----------------------------------------------------------------------------------------------------
template <bool BF16>
__global__ void __launch_bounds__(kHeadWarps * 32)
dib_int16_head1_kernel(const uint16_t* __restrict__ g, int ldg, int K, const float* __restrict__ Wc, const float* __restrict__ bc,
                       int out_act, int hid_act, float alpha, int loss, const float* __restrict__ y, long long n,
                       float inv_batch, float gscale, uint16_t* __restrict__ dg, int lddg, float* __restrict__ user_pred,
                       float* __restrict__ wpart, int wpart_stride, float* __restrict__ loss_part, float* __restrict__ acc_part) {
  constexpr int KPT = 8, ROWS = 8;
  __shared__ float red[kHeadWarps][KPT * 32];
  __shared__ float sred[kHeadWarps];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int gw = blockIdx.x * kHeadWarps + warp, nw = gridDim.x * kHeadWarps;
  float w[KPT], dw[KPT], dbh[KPT];
#pragma unroll
  for (int i = 0; i < KPT; ++i) { w[i] = Wc[lane * KPT + i]; dw[i] = 0.f; dbh[i] = 0.f; }
  const float bias = bc[0];
  float db = 0.f, lsum = 0.f, asum = 0.f;
  const bool train = dg != nullptr;
  const int myr = lane & (ROWS - 1);

  for (long long row0 = (long long)gw * ROWS; row0 < n; row0 += (long long)nw * ROWS) {
    float h[ROWS][KPT], s[ROWS];
#pragma unroll
    for (int rr = 0; rr < ROWS; ++rr) {
      const long long row = row0 + rr < n ? row0 + rr : n - 1;
      const uint4 v = *reinterpret_cast<const uint4*>(g + row * ldg + lane * KPT);
      unpack_h2<BF16>(v.x, h[rr][0], h[rr][1]); unpack_h2<BF16>(v.y, h[rr][2], h[rr][3]);
      unpack_h2<BF16>(v.z, h[rr][4], h[rr][5]); unpack_h2<BF16>(v.w, h[rr][6], h[rr][7]);
      float a = 0.f;
#pragma unroll
      for (int i = 0; i < KPT; ++i) a = fmaf(h[rr][i], w[i], a);
      s[rr] = a;
    }
    // transposing butterfly: afterwards lane L holds the warp total of s[L & 7]
#pragma unroll
    for (int o = 4; o >= 1; o >>= 1) {
#pragma unroll
      for (int i = 0; i < o; ++i) {
        const bool up = (lane & o) != 0;
        const float send = up ? s[i] : s[i + o], keep = up ? s[i + o] : s[i];
        s[i] = keep + __shfl_xor_sync(0xffffffffu, send, o);
      }
    }
    float z = s[0];
    z += __shfl_xor_sync(0xffffffffu, z, 8);
    z += __shfl_xor_sync(0xffffffffu, z, 16);
    // ---- lane L: compiled loss / metric / d loss / d z of row row0 + (L & 7)
    const long long mrow = row0 + myr;
    const bool live = mrow < n;
    z = dib_act(out_act, z + bias, alpha);
    float dz = 0.f;
    if (live && y) {
      const float t = y[mrow];
      float l;
      if (loss == DIB_LOSS_BCE_LOGITS) { l = fmaxf(z, 0.f) - z * t + log1pf(expf(-fabsf(z))); dz = 1.f / (1.f + expf(-z)) - t; }
      else if (loss == DIB_LOSS_BCE_PROBS) {
        const float ep = 1e-7f, pc = fminf(fmaxf(z, ep), 1.f - ep);
        l = -(t * logf(pc + ep) + (1.f - t) * logf(1.f - pc + ep));
        dz = (z > ep && z < 1.f - ep) ? -t / (pc + ep) + (1.f - t) / (1.f - pc + ep) : 0.f;
      } else if (loss == DIB_LOSS_SPARSE_CE_LOGITS) { l = 0.f; dz = 0.f; }        // one class: the softmax is constant
      else { const float d = z - t; l = d * d; dz = 2.f * d; }
      const float acc = loss == DIB_LOSS_SPARSE_CE_LOGITS ? ((int)t == 0 ? 1.f : 0.f) : (((z > 0.5f ? 1.f : 0.f) == t) ? 1.f : 0.f);
      if (lane < ROWS) { lsum += l; asum += acc; }
    }
    if (user_pred && live && lane < ROWS) user_pred[mrow] = z;
    if (train) {
      dz = live ? dz * inv_batch * dib_act_grad(out_act, z, alpha) : 0.f;
      if (lane < ROWS) db += dz;
#pragma unroll
      for (int rr = 0; rr < ROWS; ++rr) {
        const float dzr = __shfl_sync(0xffffffffu, dz, rr);
        if (row0 + rr >= n) break;
        const float ds = dzr * gscale;
        float d[KPT];
#pragma unroll
        for (int i = 0; i < KPT; ++i) {
          dw[i] = fmaf(h[rr][i], dzr, dw[i]);
          d[i] = ds * w[i] * dib_act_grad(hid_act, h[rr][i], alpha);
          dbh[i] += d[i];
        }
        *reinterpret_cast<uint4*>(dg + (row0 + rr) * lddg + lane * KPT) =
            make_uint4(pack_h2<BF16>(d[0], d[1]), pack_h2<BF16>(d[2], d[3]), pack_h2<BF16>(d[4], d[5]), pack_h2<BF16>(d[6], d[7]));
      }
    }
  }
  // ---- per-block partials, fixed order over the block's warps (layout as the generic kernel: [dWc | dbc | colsum dg])
  if (train) {
#pragma unroll
    for (int i = 0; i < KPT; ++i) red[warp][lane * KPT + i] = dw[i];
    __syncthreads();
    if (warp == 0) {
#pragma unroll
      for (int i = 0; i < KPT; ++i) {
        float a = 0.f;
        for (int ww = 0; ww < kHeadWarps; ++ww) a += red[ww][lane * KPT + i];
        wpart[(long long)blockIdx.x * wpart_stride + lane * KPT + i] = a;
      }
    }
    __syncthreads();
#pragma unroll
    for (int i = 0; i < KPT; ++i) red[warp][lane * KPT + i] = dbh[i];
    __syncthreads();
    if (warp == 0) {
#pragma unroll
      for (int i = 0; i < KPT; ++i) {
        float a = 0.f;
        for (int ww = 0; ww < kHeadWarps; ++ww) a += red[ww][lane * KPT + i];
        wpart[(long long)blockIdx.x * wpart_stride + (long long)K + 1 + lane * KPT + i] = a;
      }
    }
    __syncthreads();
    db = dib_warp_sum(db);
    if (lane == 0) sred[warp] = db;
    __syncthreads();
    if (threadIdx.x == 0) { float a = 0.f; for (int ww = 0; ww < kHeadWarps; ++ww) a += sred[ww]; wpart[(long long)blockIdx.x * wpart_stride + K] = a; }
    __syncthreads();
  }
  lsum = dib_warp_sum(lsum);
  if (lane == 0) sred[warp] = lsum;
  __syncthreads();
  if (threadIdx.x == 0) { float a = 0.f; for (int ww = 0; ww < kHeadWarps; ++ww) a += sred[ww]; loss_part[blockIdx.x] = a; }
  __syncthreads();
  asum = dib_warp_sum(asum);
  if (lane == 0) sred[warp] = asum;
  __syncthreads();
  if (threadIdx.x == 0) { float a = 0.f; for (int ww = 0; ww < kHeadWarps; ++ww) a += sred[ww]; acc_part[blockIdx.x] = a; }
}

template <bool BF16>
__global__ void dib_f32_to_16_kernel(const float* __restrict__ src, uint16_t* __restrict__ dst, long long n) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) {
    if constexpr (BF16) { const __nv_bfloat16 b = __float2bfloat16_rn(src[i]); dst[i] = *reinterpret_cast<const uint16_t*>(&b); }
    else { const __half b = __float2half_rn(src[i]); dst[i] = *reinterpret_cast<const uint16_t*>(&b); }
  }
}

typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                  const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                  CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
EncodeTiledFn encode_fn3() {
  static EncodeTiledFn fn = nullptr;
  if (!fn) {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) == cudaSuccess && q == cudaDriverEntryPointSuccess)
      fn = reinterpret_cast<EncodeTiledFn>(p);
  }
  return fn;
}
// K-major: [rows x ld] fp16, box 64 cols x brows
bool map_k(CUtensorMap* m, const void* base, long long cols, long long rows, long long ld, int brows) {
  cuuint64_t dims[2] = {(cuuint64_t)cols, (cuuint64_t)rows};
  cuuint64_t strides[1] = {(cuuint64_t)ld * 2};
  cuuint32_t box[2] = {64, (cuuint32_t)brows}, es[2] = {1, 1};
  return encode_fn3()(m, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 2, const_cast<void*>(base), dims, strides, box, es,
                      CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                      CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) == CUDA_SUCCESS;
}
// MN-major: [krows x ld] fp16 whose contiguous dim is M/N -> (64, krow, panel), box 64 x 64 x npanels => smem [panel][krow][128 B]
bool map_mn(CUtensorMap* m, const void* base, long long cols, long long krows, long long ld, int npanels) {
  cuuint64_t dims[3] = {64, (cuuint64_t)krows, (cuuint64_t)(cols / 64)};
  cuuint64_t strides[2] = {(cuuint64_t)ld * 2, 128};
  cuuint32_t box[3] = {64, (cuuint32_t)kBK, (cuuint32_t)npanels}, es[3] = {1, 1, 1};
  return encode_fn3()(m, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 3, const_cast<void*>(base), dims, strides, box, es,
                      CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                      CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) == CUDA_SUCCESS;
}

int g_num_sms16 = 0;
int num_sms16() {
  if (!g_num_sms16) { int dev = 0; cudaGetDevice(&dev); cudaDeviceGetAttribute(&g_num_sms16, cudaDevAttrMultiProcessorCount, dev); }
  return g_num_sms16;
}

constexpr int kGemmSmem = kStages * kStageBytes + 128 + 1024;

// streamed launch: persistent grid of at most two CTAs per SM over `ntile` tiles (one or two problems)
template <int MODE, bool BF16>
cudaError_t launch16(const CUtensorMap& mA, const CUtensorMap& mB, const Int16Args& a, const CUtensorMap& mA2, const CUtensorMap& mB2,
                     const Int16Args& a2, long long ntile, cudaStream_t st) {
  if (ntile <= 0) return cudaSuccess;
  const long long cap = 2ll * num_sms16();
  static bool attr = false;
  if (!attr) {
    cudaError_t e = cudaFuncSetAttribute(dib_int16_gemm_kernel<MODE, BF16, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, kGemmSmem);
    if (e != cudaSuccess) return e;
    attr = true;
  }
  dib_int16_gemm_kernel<MODE, BF16, false><<<(unsigned)(ntile < cap ? ntile : cap), kGemmThreads, kGemmSmem, st>>>(mA, mB, a, mA2, mB2, a2, 0);
  dib_note_launch();
  return cudaGetLastError();
}

template <int MODE, bool BF16>
cudaError_t launch16(const CUtensorMap& mA, const CUtensorMap& mB, const Int16Args& a, long long ntile, cudaStream_t st) {
  Int16Args none{};
  return launch16<MODE, BF16>(mA, mB, a, mA, mB, none, ntile, st);
}

int rb_smem(int nkb) { return nkb * kBBytes + kRbStages * kABytes + 128 + 1024; }

// resident-B launch: grid = a multiple of the column-tile count, at most one CTA per SM
template <int MODE, bool BF16>
cudaError_t launch_rb(const CUtensorMap& mA, const CUtensorMap& mB, const Int16Args& a, int nkb, cudaStream_t st) {
  const int tiles_r = DIB_CEIL_DIV(a.M, kBM), tiles_c = DIB_CEIL_DIV(a.C, kBN);
  long long grid = (long long)tiles_r * tiles_c;
  const long long cap = (long long)(num_sms16() / tiles_c) * tiles_c;
  if (grid > cap) grid = cap;
  if (grid <= 0) return cudaSuccess;
  const int smem = rb_smem(nkb);
  static int attr_smem = 0;
  if (attr_smem < smem) {
    cudaError_t e = cudaFuncSetAttribute(dib_int16_gemm_kernel<MODE, BF16, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
    if (e != cudaSuccess) return e;
    attr_smem = smem;
  }
  Int16Args none{};
  CUtensorMap mnone = mA;
  dib_int16_gemm_kernel<MODE, BF16, true><<<(unsigned)grid, kGemmThreads, smem, st>>>(mA, mB, a, mnone, mnone, none, nkb);
  dib_note_launch();
  return cudaGetLastError();
}

// the resident-B kernel applies when the [T x 128] weight slice and its A ring fit in shared memory
bool rb_ok(int T, int C) {
  if (!dib_int16_rb_enabled() || T % kBK != 0 || C % 64 != 0) return false;
  return rb_smem(T / kBK) + (int)sizeof(float) * (kConsumers / 32) * kBN <= 227 * 1024;
}

}  // namespace

static int g_int16_head1 = 1;           // single-output head: 8-rows-per-pass kernel (1, default) or the generic one (0)
int dib_int16_head1_enabled() { return g_int16_head1; }
void dib_int16_head1_set(int on) { g_int16_head1 = on ? 1 : 0; }

int g_int16_dbg = 0;
void dib_int16_dbg_set(int v) { g_int16_dbg = v; }

static int g_int16_rb = -1;
int dib_int16_rb_enabled() {
  // off by default: an A/B variant (DIB_INT16_RB=1, dib_debug_set_variant(1, 1)) that keeps the weight slice in shared memory
  // instead of re-reading it from L2 for every row tile, at one CTA per SM instead of two
  if (g_int16_rb < 0) { const char* e = getenv("DIB_INT16_RB"); g_int16_rb = (e && e[0] == '1') ? 1 : 0; }
  return g_int16_rb;
}
void dib_int16_rb_set(int on) { g_int16_rb = on ? 1 : 0; }

namespace {
struct ConvSegs { const float* src[8]; uint16_t* dst[8]; long long first[9]; int nseg; };
template <bool BF16>
__global__ void dib_f32_to_16_segs_kernel(const ConvSegs A) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= A.first[A.nseg]) return;
  int k = 0;
#pragma unroll
  for (int q = 1; q < 8; ++q) if (q < A.nseg && i >= A.first[q]) k = q;
  const float v = A.src[k][i - A.first[k]];
  uint16_t o;
  if constexpr (BF16) { const __nv_bfloat16 b = __float2bfloat16_rn(v); o = *reinterpret_cast<const uint16_t*>(&b); }
  else { const __half b = __float2half_rn(v); o = *reinterpret_cast<const uint16_t*>(&b); }
  A.dst[k][i - A.first[k]] = o;
}
}  // namespace

// several fp32 -> 16-bit conversions (the integration network's weight matrices) in one launch
cudaError_t dib_int16_convert_many(const float* const* src, void* const* dst16, const long long* n, int count, int bf16, cudaStream_t st) {
  for (int base = 0; base < count; base += 8) {
    ConvSegs A{};
    long long tot = 0; int m = 0;
    for (int k = base; k < count && m < 8; ++k) {
      if (n[k] <= 0) continue;
      A.src[m] = src[k]; A.dst[m] = static_cast<uint16_t*>(dst16[k]); A.first[m] = tot; tot += n[k]; ++m;
    }
    A.first[m] = tot; A.nseg = m;
    for (int q = m + 1; q < 9; ++q) A.first[q] = tot;
    if (m == 0) continue;
    if (bf16) dib_f32_to_16_segs_kernel<true><<<(unsigned)((tot + 255) / 256), 256, 0, st>>>(A);
    else dib_f32_to_16_segs_kernel<false><<<(unsigned)((tot + 255) / 256), 256, 0, st>>>(A);
    dib_note_launch();
  }
  return cudaGetLastError();
}

cudaError_t dib_int16_convert(const float* src, void* dst16, long long n, int bf16, cudaStream_t st) {
  if (n <= 0) return cudaSuccess;
  if (bf16) dib_f32_to_16_kernel<true><<<(unsigned)((n + 255) / 256), 256, 0, st>>>(src, static_cast<uint16_t*>(dst16), n);
  else dib_f32_to_16_kernel<false><<<(unsigned)((n + 255) / 256), 256, 0, st>>>(src, static_cast<uint16_t*>(dst16), n);
  dib_note_launch();
  return cudaGetLastError();
}

// g_out[M x N] = act(g_in[M x K] W16[K x N] + bias)
cudaError_t dib_int16_fwd(const void* g_in, int ld_in, const void* w16, const float* bias, void* g_out, int ld_out, int M,
                          int K, int N, int act, float alpha, int bf16, cudaStream_t st) {
  if (!encode_fn3()) return cudaErrorNotSupported;
  CUtensorMap mA, mB;
  if (!map_k(&mA, g_in, K, M, ld_in, kBM) || !map_mn(&mB, w16, N, K, N, kBN / 64))
    return cudaErrorInvalidValue;
  Int16Args a{};
  a.dbg = g_int16_dbg;
  a.out16 = static_cast<uint16_t*>(g_out); a.ldc = ld_out; a.bias = bias; a.M = M; a.T = K; a.C = N; a.act = act; a.alpha = alpha;
  a.out_scale = 1.f; a.nsplit = 1;
  if (rb_ok(K, N))          // weights resident in shared memory, activations streamed
    return bf16 ? launch_rb<DIB_GEMM_FWD, true>(mA, mB, a, K / kBK, st) : launch_rb<DIB_GEMM_FWD, false>(mA, mB, a, K / kBK, st);
  const long long nt = (long long)DIB_CEIL_DIV(M, kBM) * DIB_CEIL_DIV(N, kBN);
  return bf16 ? launch16<DIB_GEMM_FWD, true>(mA, mB, a, nt, st) : launch16<DIB_GEMM_FWD, false>(mA, mB, a, nt, st);
}

// dz_in[M x K] = (dz[M x N] W16[K x N]^T) * act'(g_in[M x K])      (g_in may be null: no activation, e.g. d_emb)
cudaError_t dib_int16_dgrad(const void* dz, int ld_dz, const void* w16, const void* g_in, int ld_g, void* dz_in, int ld_out,
                            int M, int K, int N, int act, float alpha, float* colsum_part, int bf16, cudaStream_t st) {
  if (!encode_fn3()) return cudaErrorNotSupported;
  CUtensorMap mA, mB;
  if (!map_k(&mA, dz, N, M, ld_dz, kBM) || !map_k(&mB, w16, N, K, N, kBN))
    return cudaErrorInvalidValue;
  Int16Args a{};
  a.dbg = g_int16_dbg;
  a.out16 = static_cast<uint16_t*>(dz_in); a.ldc = ld_out; a.X = static_cast<const uint16_t*>(g_in); a.ldx = ld_g;
  a.M = M; a.T = N; a.C = K; a.act = act; a.alpha = alpha; a.out_scale = 1.f; a.nsplit = 1; a.dbias = colsum_part;
  if (rb_ok(N, K))          // W^T slice resident, dz streamed
    return bf16 ? launch_rb<DIB_GEMM_DGRAD, true>(mA, mB, a, N / kBK, st) : launch_rb<DIB_GEMM_DGRAD, false>(mA, mB, a, N / kBK, st);
  const long long nt = (long long)DIB_CEIL_DIV(M, kBM) * DIB_CEIL_DIV(K, kBN);
  return bf16 ? launch16<DIB_GEMM_DGRAD, true>(mA, mB, a, nt, st) : launch16<DIB_GEMM_DGRAD, false>(mA, mB, a, nt, st);
}

// dW[K x N] (fp32 split partials, * out_scale) = g_in[M x K]^T dz[M x N];  db = colsum dz
cudaError_t dib_int16_wgrad(const void* g_in, int ld_g, const void* dz, int ld_dz, float* dW_part, float* db_part, int M, int K,
                            int N, int nsplit, int rows_per_split, long long split_stride, float out_scale, int bf16, cudaStream_t st) {
  if (!encode_fn3()) return cudaErrorNotSupported;
  CUtensorMap mA, mB;
  if (!map_mn(&mA, g_in, K, M, ld_g, kBM / 64) || !map_mn(&mB, dz, N, M, ld_dz, kBN / 64))
    return cudaErrorInvalidValue;
  Int16Args a{};
  a.dbg = g_int16_dbg;
  a.out32 = dW_part; a.ldc = N; a.dbias = nullptr; a.M = M; a.T = 0; a.C = N; a.R = K; a.out_scale = out_scale;
  a.nsplit = nsplit; a.rows_per_split = rows_per_split; a.split_stride = split_stride;
  (void)db_part;   // bias gradients come from the kernel that PRODUCES dz (dgrad epilogue / output head), not from here
  const long long nt = (long long)DIB_CEIL_DIV(N, kBN) * DIB_CEIL_DIV(K, kBM) * nsplit;
  return bf16 ? launch16<DIB_GEMM_WGRAD, true>(mA, mB, a, nt, st) : launch16<DIB_GEMM_WGRAD, false>(mA, mB, a, nt, st);
}

static int g_int16_fwd2 = -1;            // fused [hidden, hidden, head] kernel for single-output models (1, default) or the separate kernels (0)
int dib_int16_fwd2_enabled() {
  if (g_int16_fwd2 < 0) { const char* e = getenv("DIB_INT16_FWD2"); g_int16_fwd2 = (e && e[0] == '0') ? 0 : 1; }
  return g_int16_fwd2;
}
void dib_int16_fwd2_set(int on) { g_int16_fwd2 = on ? 1 : 0; }
int dib_int16_fwd2_ok(int K0, int N1, int N2, int out_dim) {
  return dib_int16_fwd2_enabled() && K0 % kBK == 0 && K0 >= kBK && N1 == kF2N && N2 == kF2N && out_dim == 1;
}

// g1 = act(g_in W0 + b0) -> HBM;  g2 = act(g1 W1 + b1) (on chip);  logit = g2 . wout + bout;  compiled loss / metric;
// training (dg2 != null): dg2, per-CTA partials of the output layer's gradients and of the last hidden layer's bias gradient.
// *nblocks = CTAs launched = rows of wpart / loss_part / acc_part written.
cudaError_t dib_int16_fwd2_head(const void* g_in, int ld_in, int K0, const void* w16_0, const float* b0, const void* w16_1, const float* b1,
                                void* g1, const float* wout, const float* bout, int act, int out_act, float alpha, int loss, const float* y,
                                int M, float inv_batch, float gscale, void* dg2, float* user_pred, float* wpart, int wpart_stride,
                                float* loss_part, float* acc_part, int* nblocks, int bf16, cudaStream_t st) {
  if (!encode_fn3()) return cudaErrorNotSupported;
  CUtensorMap mA, mW0, mW1;
  if (!map_k(&mA, g_in, K0, M, ld_in, kBM) || !map_mn(&mW0, w16_0, kF2N, K0, kF2N, kF2N / 64) || !map_mn(&mW1, w16_1, kF2N, kF2N, kF2N, kF2N / 64))
    return cudaErrorInvalidValue;
  Fwd2Args a{};
  a.b0 = b0; a.b1 = b1; a.wout = wout; a.bout = bout; a.g1 = static_cast<uint16_t*>(g1); a.ldg1 = kF2N;
  a.dg2 = static_cast<uint16_t*>(dg2); a.lddg = kF2N; a.y = y; a.user_pred = user_pred; a.wpart = wpart; a.wpart_stride = wpart_stride;
  a.loss_part = loss_part; a.acc_part = acc_part; a.M = M; a.nk0 = K0 / kBK; a.act = act; a.out_act = out_act; a.loss = loss;
  a.alpha = alpha; a.inv_batch = inv_batch; a.gscale = gscale;
  const int tiles = DIB_CEIL_DIV(M, kBM);
  const int grid = tiles < num_sms16() ? tiles : num_sms16();
  *nblocks = grid;
  if (grid <= 0) return cudaSuccess;
  cudaError_t e = cudaErrorInvalidValue;
#define DIB_F2_LAUNCH(BF, ACT)                                                                                                       \
  do {                                                                                                                               \
    static bool attr = false;                                                                                                        \
    e = attr ? cudaSuccess : cudaFuncSetAttribute(dib_int16_fwd2_kernel<BF, ACT>, cudaFuncAttributeMaxDynamicSharedMemorySize, kF2Smem); \
    if (e != cudaSuccess) return e;                                                                                                  \
    attr = true;                                                                                                                     \
    dib_int16_fwd2_kernel<BF, ACT><<<grid, kF2Threads, kF2Smem, st>>>(mA, mW0, mW1, a);                                               \
  } while (0)
#define DIB_F2_ACT(ACT) do { if (bf16) DIB_F2_LAUNCH(true, ACT); else DIB_F2_LAUNCH(false, ACT); } while (0)
  switch (act) {
    case DIB_ACT_LINEAR: DIB_F2_ACT(DIB_ACT_LINEAR); break;
    case DIB_ACT_RELU: DIB_F2_ACT(DIB_ACT_RELU); break;
    case DIB_ACT_TANH: DIB_F2_ACT(DIB_ACT_TANH); break;
    case DIB_ACT_LEAKY_RELU: DIB_F2_ACT(DIB_ACT_LEAKY_RELU); break;
    case DIB_ACT_SIGMOID: DIB_F2_ACT(DIB_ACT_SIGMOID); break;
    case DIB_ACT_ELU: DIB_F2_ACT(DIB_ACT_ELU); break;
    default: return cudaErrorInvalidValue;
  }
#undef DIB_F2_ACT
#undef DIB_F2_LAUNCH
  dib_note_launch();
  return cudaGetLastError();
}

// the weight gradients of TWO layers in one launch (same batch M, same partial stride): dW_j = g_in_j^T dz_j over batch slices
cudaError_t dib_int16_wgrad_pair(const void* g_in0, int K0, const void* dz0, int N0, float* dW_part0, int nsplit0, int rps0,
                                 const void* g_in1, int K1, const void* dz1, int N1, float* dW_part1, int nsplit1, int rps1,
                                 int M, long long split_stride, float out_scale, int bf16, cudaStream_t st) {
  if (!encode_fn3()) return cudaErrorNotSupported;
  CUtensorMap mA, mB, mA2, mB2;
  if (!map_mn(&mA, g_in0, K0, M, K0, kBM / 64) || !map_mn(&mB, dz0, N0, M, N0, kBN / 64) ||
      !map_mn(&mA2, g_in1, K1, M, K1, kBM / 64) || !map_mn(&mB2, dz1, N1, M, N1, kBN / 64))
    return cudaErrorInvalidValue;
  Int16Args a{}, b{};
  a.dbg = b.dbg = g_int16_dbg;
  a.out32 = dW_part0; a.ldc = N0; a.M = M; a.C = N0; a.R = K0; a.out_scale = out_scale; a.nsplit = nsplit0; a.rows_per_split = rps0; a.split_stride = split_stride;
  b.out32 = dW_part1; b.ldc = N1; b.M = M; b.C = N1; b.R = K1; b.out_scale = out_scale; b.nsplit = nsplit1; b.rows_per_split = rps1; b.split_stride = split_stride;
  const long long nt = (long long)DIB_CEIL_DIV(K0, kBM) * DIB_CEIL_DIV(N0, kBN) * nsplit0 + (long long)DIB_CEIL_DIV(K1, kBM) * DIB_CEIL_DIV(N1, kBN) * nsplit1;
  return bf16 ? launch16<DIB_GEMM_WGRAD, true>(mA, mB, a, mA2, mB2, b, nt, st) : launch16<DIB_GEMM_WGRAD, false>(mA, mB, a, mA2, mB2, b, nt, st);
}

int dib_int16_head_blocks(int num_sms) { return num_sms * 2; }

cudaError_t dib_int16_head(const void* g, int ldg, int K, const float* Wc, const float* bc, int out_dim, int out_act, int hid_act,
                           float alpha, int loss, const float* y, long long n, float inv_batch, float gscale, void* dg, int lddg,
                           float* user_pred, float* wpart, int wpart_stride, float* loss_part, float* acc_part, int nblocks,
                           int bf16, cudaStream_t st) {
  if (out_dim > kHeadMaxOut || out_dim < 1 || K != 256) return cudaErrorInvalidValue;
#define DIB_HEAD_T(OUT, BF)                                                                                             \
  dib_int16_head_kernel<8, OUT, (OUT <= 2 ? 4 : 1), BF><<<nblocks, kHeadWarps * 32, 0, st>>>(static_cast<const uint16_t*>(g), ldg, K, Wc, bc, out_dim,  \
      out_act, hid_act, alpha, loss, y, n, inv_batch, gscale, static_cast<uint16_t*>(dg), lddg, user_pred, wpart, wpart_stride, \
      loss_part, acc_part)
#define DIB_HEAD(OUT) do { if (bf16) DIB_HEAD_T(OUT, true); else DIB_HEAD_T(OUT, false); } while (0)
  if (out_dim == 1 && dib_int16_head1_enabled()) {
    if (bf16) dib_int16_head1_kernel<true><<<nblocks, kHeadWarps * 32, 0, st>>>(static_cast<const uint16_t*>(g), ldg, K, Wc, bc, out_act,
        hid_act, alpha, loss, y, n, inv_batch, gscale, static_cast<uint16_t*>(dg), lddg, user_pred, wpart, wpart_stride, loss_part, acc_part);
    else dib_int16_head1_kernel<false><<<nblocks, kHeadWarps * 32, 0, st>>>(static_cast<const uint16_t*>(g), ldg, K, Wc, bc, out_act,
        hid_act, alpha, loss, y, n, inv_batch, gscale, static_cast<uint16_t*>(dg), lddg, user_pred, wpart, wpart_stride, loss_part, acc_part);
  } else if (out_dim == 1) DIB_HEAD(1);
  else if (out_dim == 2) DIB_HEAD(2);
  else if (out_dim <= 4) DIB_HEAD(4);
  else if (out_dim <= 8) DIB_HEAD(8);
  else DIB_HEAD(16);
#undef DIB_HEAD
#undef DIB_HEAD_T
  dib_note_launch();
  return cudaGetLastError();
}
