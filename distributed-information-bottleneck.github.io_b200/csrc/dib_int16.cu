// dib_int16.cu -- the integration network (models.py:81-84,122) in the tensor-core mode: 16-bit activations in HBM
// (emb, g_k, dz_k as fp16 -> half the traffic of the fp32 layout), wgmma on 16-bit operands with fp32 accumulation.
//
//   * dib_int16_gemm_kernel<MODE>: TMA-fed, mbarrier-pipelined 128 x 128 tile GEMM (K step 64 = one 128-byte swizzle
//     span) with fused epilogues:  FWD  g = act(A W + b) -> fp16;  DGRAD  dz_in = (dz W^T) * act'(g_in) -> fp16 and the
//     column sums of dz_in (bias gradient of the layer below);  WGRAD  dW = g^T dz over a batch slice -> fp32 split partial
//     (scaled back by 1/S).
//   * dib_int16_head_kernel: the narrow output layer (out <= 16) fused with everything around it -- logits, compiled
//     loss + accuracy, d loss / d logits, the dgrad into the last hidden layer (incl. its act') and the output layer's
//     own weight/bias gradients -- one pass over the last hidden activation.  dib_int16_head1_kernel: the same for out = 1.
//   * dib_int16_fwd2_kernel: the last two 256-wide hidden layers and the single-output head of models with out = 1, and in
//     training the dgrad chain below the head: down to the 16-bit embedding gradient, or to the first fused layer's
//     pre-activation gradient when another hidden layer lies below it.
// Which tail and which head kernel run is the caller's choice (the model handle's route in dib_api.cu); nothing here
// reads process-wide state.
// Gradient operands are scaled by the power-of-two loss scale S (see dib_enc_fused.cu) to stay inside fp16 range.
//
// The GEMM kernels are warp-specialised: warps 0..7 are two consumer warpgroups (warpgroup g computes rows [64 g, 64 g + 64)
// of the 128-row tile with m64nNk16 wgmma instructions, accumulators in registers, and runs the epilogue), warp 8 issues
// the TMA loads of the shared-memory ring.
#include <cuda.h>
#include <cuda_bf16.h>
#include <cuda_fp16.h>

#include <type_traits>

#include "dib_common.cuh"
#include "dib_kernels.h"
#include "dib_sm90.cuh"

namespace {

using namespace sm90;

constexpr int kBM = 128, kBN = 128, kBK = 64, kStages = 3;
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
__device__ __forceinline__ uint32_t ld_shared_b32(uint32_t addr) {
  uint32_t v;
  asm volatile("ld.shared.b32 %0, [%1];" : "=r"(v) : "r"(addr) : "memory");
  return v;
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
template <int MODE, bool BF16>
__global__ void __launch_bounds__(kGemmThreads, 2)
dib_int16_gemm_kernel(const __grid_constant__ CUtensorMap mapA, const __grid_constant__ CUtensorMap mapB, const Int16Args a,
                      const __grid_constant__ CUtensorMap mapA2, const __grid_constant__ CUtensorMap mapB2, const Int16Args a2) {
  // (a2, mapA2, mapB2): an optional SECOND weight-gradient problem walked by the same launch (a2.nsplit > 0, WGRAD only): the two
  // layers' tiles together fill one wave of CTAs, which neither fills alone
  constexpr bool A_MN = (MODE == DIB_GEMM_WGRAD), B_MN = (MODE != DIB_GEMM_DGRAD);
  extern __shared__ uint8_t smem_raw[];
  const uint32_t ring = (smem_u32(smem_raw) + 1023u) & ~1023u;
  const uint32_t bar_base = ring + kStages * kStageBytes;
  auto full_bar = [&](int s) { return bar_base + 8u * s; };
  auto empty_bar = [&](int s) { return bar_base + 8u * (kStages + s); };

  __shared__ float colsum_s[kConsumers / 32][kBN];
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int R0 = (MODE == DIB_GEMM_WGRAD) ? a.R : a.M, C0 = a.C;
  const int tiles_r = DIB_CEIL_DIV(R0, kBM), tiles_c = DIB_CEIL_DIV(C0, kBN);
  const int nsp = (MODE == DIB_GEMM_WGRAD) ? a.nsplit : 1;
  const int ntile0 = tiles_r * tiles_c * nsp;
  const bool two = (MODE == DIB_GEMM_WGRAD) && a2.nsplit > 0;
  const int tiles_r2 = two ? DIB_CEIL_DIV(a2.R, kBM) : 0, tiles_c2 = two ? DIB_CEIL_DIV(a2.C, kBN) : 0;
  const int ntile = ntile0 + tiles_r2 * tiles_c2 * (two ? a2.nsplit : 0);

  int prob = 0;                                     // which problem the tile last decoded belongs to (per thread)
  auto decode = [&](int tile, int& r0, int& c0, int& split, int& t_begin, int& nk) {
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
    for (int s = 0; s < kStages; ++s) { mbar_init(full_bar(s), 1); mbar_init(empty_bar(s), kEmptyArrivals); }
    fence_barrier_init();
  }
  __syncthreads();

  if (warp == kProducerWarp) {
    // ============================================================== TMA producer (one lane)
    if (lane == 0) {
      tma_prefetch_desc(&mapA); tma_prefetch_desc(&mapB);
      if (two) { tma_prefetch_desc(&mapA2); tma_prefetch_desc(&mapB2); }
      uint32_t s = 0, ph = 0;
      for (int tile = blockIdx.x; tile < ntile; tile += gridDim.x) {
        int r0, c0, split, t_begin, nk;
        decode(tile, r0, c0, split, t_begin, nk);
        const CUtensorMap* mA = prob ? &mapA2 : &mapA;
        const CUtensorMap* mB = prob ? &mapB2 : &mapB;
        for (int k = 0; k < nk; ++k) {
          mbar_wait(empty_bar(s), ph ^ 1);
          mbar_expect_tx(full_bar(s), kStageBytes);
          const uint32_t a_dst = ring + s * kStageBytes, b_dst = a_dst + kABytes;
          const int t0 = t_begin + k * kBK;
          if constexpr (A_MN) tma_load_3d(a_dst, mA, full_bar(s), 0, t0, r0 / 64);
          else                tma_load_2d(a_dst, mA, full_bar(s), t0, r0);
          if constexpr (B_MN) tma_load_3d(b_dst, mB, full_bar(s), 0, t0, c0 / 64);
          else                tma_load_2d(b_dst, mB, full_bar(s), t0, c0);
          if (++s == kStages) { s = 0; ph ^= 1; }
        }
      }
    }
  } else {
    // ============================================================== consumer warpgroups: MMAs + epilogue
    const int wg = tid >> 7, q = lane & 3;
    const int rb = 64 * wg + 16 * (warp & 3) + (lane >> 2);       // tile row of this thread's accumulator elements
    uint32_t s = 0, ph = 0;
    for (int tile = blockIdx.x; tile < ntile; tile += gridDim.x) {
      int r0, c0, split, t_begin, nk;
      decode(tile, r0, c0, split, t_begin, nk);
      float acc[64];
#pragma unroll
      for (int i = 0; i < 64; ++i) acc[i] = 0.f;
      if (nk > 0) {
        uint32_t prev = 0;
        for (int k = 0; k < nk; ++k) {
          mbar_wait(full_bar(s), ph);
          const uint32_t a_base = ring + s * kStageBytes;
          const uint32_t b_base = a_base + kABytes;
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
          if (++s == kStages) { s = 0; ph ^= 1; }
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
            if (live)
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
            if (live) *reinterpret_cast<uint32_t*>(a.out16 + (long long)r * a.ldc + c) = pack_h2<BF16>(v0, v1);
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
//                      e0  g1 = act(D0 + b0) -> 16-bit -> swizzled shared tile (= L1's A operand) -> TMA tensor store to HBM
//                          (the weight gradients need it) while L1 reads the same tile
//                      L1  D1 = g1 W1  (W1 k-blocks through the same ring)
//                      e1  g2 = act(D1 + b1) kept PACKED IN REGISTERS, logit = g2 . w + b, compiled loss / metric,
//                          d loss / d logit, dg2 = dz w act'(g2) -> HBM, output-layer weight / bias gradients and the bias gradient
//                          of the last hidden layer as per-CTA partials.  relu / leaky relu / linear: each thread first keeps the
//                          bits g1 > 0 of its own g1 words (all that act'(g1) needs) in 4 registers, then writes dg2 over those
//                          words of the g1 tile -> TMA tensor store; other activations store dg2 from the fragments.
//   training, backward stages on (dg1 != null), the dgrad chain of the same rows:
//                      D1  acc = dg2 W1^T  (dg2 packed in registers = the wgmma A fragment; W1 K-major through the ring;
//                          two 128-column chunks)
//                      e2  dg1 = acc act'(g1) (act' from the g1 > 0 bits, or g1 read back from the shared tile) -> over the
//                          shared tile -> TMA tensor store, and packed into registers; its column sums per tile (bias
//                          gradient of the first fused layer) -> dbpart, in the order of the DGRAD epilogue
//                      D0  (only when the layer below is the embedding, which has no act') d emb = dg1 W0^T over 128-column
//                          chunks (W0 K-major through the ring)
//                      e3  16-bit d emb -> the g1 tile (free by then) -> TMA tensor store
// The tensor stores leave no partial-sector writes behind and run while the MMAs go on; 4-byte fragment stores straight
// from the accumulators stall the epilogue that issues them.  Only the dg2 of tanh / sigmoid / elu, produced while the g1
// tile still holds the g1 that e2's act' needs, leaves as fragment stores.
// g2 never reaches HBM, and the head's re-read of it (and its launch) disappears; with the backward stages, neither do
// the two dgrad launches nor their re-reads of dg2, dg1 and g1.  A warp owns 16 whole rows of the accumulator, so each
// row's logit is complete after a reduction over the 4 lanes that share the row.  Every MMA keeps the operands and the
// k order of dib_int16_dgrad, and every sum its order: the results are those of the separate launches, bit for bit.
// Ring stages of a tile: nk0 x (A, W0 MN-major), 4 x W1 MN-major; then 2 x 2 x W1 K-major and K0 / 128 x 2 x W0 K-major
// (B only: 128 output columns x 128 k each).  The ring is 3 deep, so two loads are in flight while the consumers run a
// stage's MMAs, and during each epilogue the producer fills the first stages of the next phase (or of the next tile).
// Shared memory: the 3-stage ring (3 x 48 KB), the g1 tile (4 swizzled 64-column panels of 128 rows, 64 KB), the barriers,
// and statically the bias / head-weight rows and one [8][256] column-sum scratch (used in turn by the output layer's dW,
// the bias gradient of the last hidden layer and that of the first fused layer).
// ====================================================================================================
// The warp's column sums of 8 N columns: v[2 j + e] is this thread's partial of column 8 j + 2 q + e (the sum of its two
// rows); the 8 lanes that share q add them over the same pairs of lanes, in the same order, as quad_col_sum (so every sum
// has its bits), but each step keeps only half of the columns and sends the other half to the partner: 7 N / 4 shuffles in
// three independent batches instead of 6 N in dependent chains of three.  Lane (q, b0 = lane bit 2, b1 = bit 3, b2 = bit 4)
// ends with columns 8 (4 m + 2 b2 + b1) + 2 q + b0, which it writes to col (bank 8 b1 + 16 b2 + 2 q + b0: no conflicts).
template <int N>
__device__ __forceinline__ void quad_col_sums(const float (&v)[2 * N], float* col, int lane) {
  const int q = lane & 3, b0 = (lane >> 2) & 1, b1 = (lane >> 3) & 1, b2 = (lane >> 4) & 1;
  float s1[N], s2[N / 2], s3[N / 4];
#pragma unroll
  for (int m = 0; m < N; ++m) s1[m] = (b0 ? v[2 * m + 1] : v[2 * m]) + __shfl_xor_sync(0xffffffffu, b0 ? v[2 * m] : v[2 * m + 1], 4);
#pragma unroll
  for (int m = 0; m < N / 2; ++m) s2[m] = (b1 ? s1[2 * m + 1] : s1[2 * m]) + __shfl_xor_sync(0xffffffffu, b1 ? s1[2 * m] : s1[2 * m + 1], 8);
#pragma unroll
  for (int m = 0; m < N / 4; ++m) s3[m] = (b2 ? s2[2 * m + 1] : s2[2 * m]) + __shfl_xor_sync(0xffffffffu, b2 ? s2[2 * m] : s2[2 * m + 1], 16);
#pragma unroll
  for (int m = 0; m < N / 4; ++m) col[8 * (4 * m + 2 * b2 + b1) + 2 * q + b0] = s3[m];
}

constexpr int kF2N = 256, kF2Stages = 3;
constexpr int kF2AB = kBM * 128, kF2BB = kF2N * 128, kF2Stage = kF2AB + kF2BB;      // 16 KB + 32 KB
constexpr int kF2BtN = 128, kF2BtB = kF2BtN * 128;   // backward stages: B only, two k-blocks of 128 K-major rows (2 x 16 KB)
constexpr int kF2G1Off = kF2Stages * kF2Stage;
constexpr int kF2BarOff = kF2G1Off + kBM * kF2N * 2;
constexpr int kF2Smem = kF2BarOff + 64 + 1024;
// static shared memory of the kernel: s_b0, s_b1, s_w; s_col; s_red
constexpr int kF2StaticSmem = (3 * kF2N + (kConsumers / 32) * kF2N + 3 * (kConsumers / 32)) * (int)sizeof(float);
static_assert(2 * 8 * kF2Stages <= 64, "the ring's full and empty barriers fit their 64 bytes");
static_assert(kF2Smem + kF2StaticSmem <= 232448, "fused tail: shared memory above the sm_90 227 KB per-block opt-in");

struct Fwd2Args {
  const float *b0, *b1, *wout, *bout;
  uint16_t* dg2; int lddg;            // out (training) or null: gradient w.r.t. the second fused layer's pre-activation, x gscale
  bool bwd;                           // training, backward stages: dg1, the gradient w.r.t. the first fused layer's
                                      // pre-activation [M x 256] x gscale, via mapDg1
  float* dbpart;                      // with dg1: column sums of dg1 per 128-row tile [tiles][256]
  int demb_cols;                      // with dg1, > 0: the layer below is the embedding; d emb [M x demb_cols] via mapDemb
  const float* y; float* user_pred;
  const float* wts;                   // WEIGHTED: the rows' sample weights
  float* wpart; int wpart_stride; float *loss_part, *acc_part;
  int M, nk0, act, out_act, loss;
  float alpha, inv_batch, gscale;
};

// ACT is a template parameter: the activation switch inside the fully unrolled register-resident passes would otherwise be
// evaluated per element.  WEIGHTED: row i's loss and d loss / d logit carry its sample weight a.wts[i] (in e1's loss block,
// before any 16-bit rounding); the unweighted instantiations do not read it.
constexpr int kF2Threads = kConsumers + 128;      // + a producer warpgroup, so that setmaxnreg can move its registers to the consumers
template <bool BF16, int ACT, bool WEIGHTED>
__global__ void __launch_bounds__(kF2Threads, 1)
dib_int16_fwd2_kernel(const __grid_constant__ CUtensorMap mapA, const __grid_constant__ CUtensorMap mapW0,
                      const __grid_constant__ CUtensorMap mapW1, const __grid_constant__ CUtensorMap mapW1t,
                      const __grid_constant__ CUtensorMap mapW0t, const __grid_constant__ CUtensorMap mapDemb,
                      const __grid_constant__ CUtensorMap mapG1, const __grid_constant__ CUtensorMap mapDg1,
                      const __grid_constant__ CUtensorMap mapDg2, const Fwd2Args a) {
  // relu, leaky relu and linear: act'(g1) is a function of the predicate g1 > 0 alone, so 128 bits per thread stand in for
  // its g1 words, the g1 tile is free from e1 on, and dg2 leaves through it by TMA as dg1 does
  constexpr bool kStageDg2 = ACT == DIB_ACT_RELU || ACT == DIB_ACT_LEAKY_RELU || ACT == DIB_ACT_LINEAR;
  extern __shared__ uint8_t smem_raw[];
  const uint32_t sb = (smem_u32(smem_raw) + 1023u) & ~1023u;
  const uint32_t bar_base = sb + kF2BarOff;
  auto full_bar = [&](int s) { return bar_base + 8u * s; };
  auto empty_bar = [&](int s) { return bar_base + 8u * (kF2Stages + s); };
  const uint32_t g1s = sb + kF2G1Off;

  __shared__ __align__(16) float s_b0[kF2N], s_b1[kF2N], s_w[kF2N];
  __shared__ float s_col[kConsumers / 32][kF2N];     // per-warp column sums of one quantity at a time
  __shared__ float s_red[3][kConsumers / 32];
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int ntile = DIB_CEIL_DIV(a.M, kBM);
  const bool bwd = a.bwd;

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
      if (bwd) { tma_prefetch_desc(&mapW1t); if (a.demb_cols > 0) tma_prefetch_desc(&mapW0t); }
      uint32_t s = 0, ph = 0;
      auto b_stage = [&](const CUtensorMap* m, int k0, int c0) {     // a B-only stage: 128 K-major rows x 128 k
        mbar_wait(empty_bar(s), ph ^ 1);
        mbar_expect_tx(full_bar(s), 2 * kF2BtB);
        tma_load_2d(sb + s * kF2Stage + kF2AB, m, full_bar(s), k0, c0);
        tma_load_2d(sb + s * kF2Stage + kF2AB + kF2BtB, m, full_bar(s), k0 + kBK, c0);
        if (++s == kF2Stages) { s = 0; ph ^= 1; }
      };
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
        if (bwd) {
          for (int c0 = 0; c0 < kF2N; c0 += kF2BtN)
            for (int k = 0; k < kF2N; k += 2 * kBK) b_stage(&mapW1t, k, c0);
          for (int c0 = 0; c0 < a.demb_cols; c0 += kF2BtN)
            for (int k = 0; k < kF2N; k += 2 * kBK) b_stage(&mapW0t, k, c0);
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
  // acc = A[64 x 256] B[256 x 128] over 2 B-only ring stages of two k-blocks; A packed in registers (ap[4 t .. 4 t + 3]: the
  // fragment of k16 step t).  128-column chunks: a 256-column accumulator next to the 64 A registers does not fit the
  // register budget.  Stages of 128 k: half as many stages as 64-deep ones, so half as many load latencies to hide.
  auto mainloop_rs = [&](float (&acc)[64], const uint32_t (&ap)[64]) {
    uint32_t prev = 0;
#pragma unroll
    for (int k = 0; k < kF2N / (2 * kBK); ++k) {
      mbar_wait(full_bar(s), ph);
      const uint32_t bt = sb + s * kF2Stage + kF2AB;
      wgmma_fence();
#pragma unroll
      for (int kk = 0; kk < 2 * kBK / 16; ++kk) {
        const int t = 8 * k + kk;
        const uint32_t af[4] = {ap[4 * t], ap[4 * t + 1], ap[4 * t + 2], ap[4 * t + 3]};
        wgmma_m64n128k16_rs<BF16, 0>(acc, af, desc_kmaj(bt + (kk >> 2) * kF2BtB, kk & 3), t > 0 ? 1u : 0u);
      }
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
  // this thread's word (columns c, c + 1 of row r) in the swizzled g1 tile; every thread reads back only words it wrote
  auto g1_word = [&](int c, int r) { return g1s + (c >> 6) * kF2AB + r * 128 + ((((c & 63) >> 3) ^ (r & 7)) << 4) + 4 * q; };
  // the warpgroup's tensor stores, all (N = 0) or all but the last group (N = 1), have read its rows of the g1 tile
  auto stores_drained = [&](auto n_pending) {
    if ((tid & 127) == 0) bulk_wait_read<decltype(n_pending)::value>();
    named_bar_sync(2 + wg, 128);
  };
  // the warpgroup's rows of g1-tile panels [p0, p0 + n) -> columns [c0, c0 + 64 n) of a 16-bit [M x *] tensor as one store
  // group (rows past M are not written); the caller has fenced its shared writes and synchronised the warpgroup
  auto store_panels = [&](const CUtensorMap* m, int tile, int p0, int n, int c0) {
    if ((tid & 127) == 0) {
      for (int p = 0; p < n; ++p) tma_store_2d(m, g1s + (p0 + p) * kF2AB + wg * 64 * 128, c0 + 64 * p, tile * kBM + 64 * wg);
      bulk_commit();
    }
  };

  for (int tile = blockIdx.x; tile < ntile; tile += gridDim.x) {
    const long long row_lo = (long long)tile * kBM + rb;
    float acc[128];
#pragma unroll
    for (int i = 0; i < 128; ++i) acc[i] = 0.f;
    // ---------------- L0, e0: g1 = act(D0 + b0) -> shared tile (L1's A operand) -> HBM
    mainloop(acc, a.nk0, true);
    stores_drained(std::integral_constant<int, 0>());   // the previous tile's stores have read the g1 tile
#pragma unroll
    for (int j = 0; j < kF2N / 8; ++j) {
      const int c = 8 * j + 2 * q;
      const float2 bv = *reinterpret_cast<const float2*>(&s_b0[c]);
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const uint32_t w = pack_h2<BF16>(dib_act16(ACT, acc[4 * j + 2 * h] + bv.x, a.alpha), dib_act16(ACT, acc[4 * j + 2 * h + 1] + bv.y, a.alpha));
        st_shared_b32(g1_word(c, rb + 8 * h), w);
      }
    }
    fence_proxy_async_smem();
    named_bar_sync(2 + wg, 128);                     // this warpgroup's rows of g1 are complete
    store_panels(&mapG1, tile, 0, kF2N / 64, 0);
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
        // an opaque copy: else the compiler keeps these unpacked floats (twice the registers of g2p) alive for pass 2 instead
        // of unpacking g2p again there, and spills once pass 2 feeds the backward stages
        uint32_t pc;
        asm("mov.b32 %0, %1;" : "=r"(pc) : "r"(p));
        float h0, h1;
        unpack_h2<BF16>(pc, h0, h1);
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
      float dz = 0.f, ib = a.inv_batch;
      if (live && a.y) {
        const float t = a.y[row];
        float wr = 1.f;
        if constexpr (WEIGHTED) { wr = a.wts[row]; ib *= wr; }
        float l = -0.f, acc1 = -0.f;
        if (a.loss == DIB_LOSS_SPARSE_CE_LOGITS) {   // one class: the softmax is constant; an invalid label gives NaN
          l = dz = dib_sparse_label(t, 1) < 0 ? __int_as_float(0x7fc00000) : 0.f;
          acc1 = t == 0.f ? 1.f : 0.f;
        }
        else dz = dib_loss_add_t<WEIGHTED>(a.loss, z, t, wr, l, acc1);
        if (q == 0) { lsum += l; asum += acc1; }
      }
      if (a.user_pred && live && q == 0) a.user_pred[row] = z;
      dzs[h] = live ? dz * ib * dib_act_grad(a.out_act, z, a.alpha) : 0.f;
      ds[h] = dzs[h] * a.gscale;
      if (q == 0) dbo += dzs[h];
    }
    // kStageDg2: bit 4 (j & 7) + 2 h + e of g1m[j / 8] is g1 > 0 for half e of this thread's g1 word (8 j + 2 q, rb + 8 h)
    uint32_t g1m[4] = {0u, 0u, 0u, 0u};
    if (train) {
      // ---------------- e1, pass 2: column sums of g2 dz (output-layer dW).  The 8 warps cover the tile's 128 rows: fixed-order
      // combine into the thread-owned column
      {
        float cw[kF2N / 4];
#pragma unroll
        for (int j = 0; j < kF2N / 8; ++j) {
          cw[2 * j] = cw[2 * j + 1] = 0.f;
#pragma unroll
          for (int h = 0; h < 2; ++h) {
            float h0, h1;
            unpack_h2<BF16>(g2p[2 * j + h], h0, h1);
            cw[2 * j] += h0 * dzs[h]; cw[2 * j + 1] += h1 * dzs[h];
          }
        }
        quad_col_sums<kF2N / 8>(cw, s_col[warp], lane);
      }
      named_bar_sync(1, kConsumers);
#pragma unroll
      for (int w = 0; w < kConsumers / 32; ++w) acc_dw += s_col[w][tid];
      named_bar_sync(1, kConsumers);
      // ---------------- e1, pass 3: dg2 = ds w act'(g2) -> HBM and packed into g2p (A of D1); its column sums (bias gradient).
      // kStageDg2: each packed dg2 word first takes the place of the thread's g1 word of the same position (its g1 > 0 bits go
      // to g1m), then the tile leaves as one tensor store group
      if constexpr (kStageDg2) stores_drained(std::integral_constant<int, 0>());   // the g1 store has read the tile
      float cb[kF2N / 4];
#pragma unroll
      for (int j = 0; j < kF2N / 8; ++j) {
        const int c = 8 * j + 2 * q;
        const float2 wv = *reinterpret_cast<const float2*>(&s_w[c]);
        cb[2 * j] = cb[2 * j + 1] = 0.f;
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          float h0, h1;
          unpack_h2<BF16>(g2p[2 * j + h], h0, h1);
          const float d0 = ds[h] * wv.x * dib_act_grad(ACT, h0, a.alpha), d1 = ds[h] * wv.y * dib_act_grad(ACT, h1, a.alpha);
          cb[2 * j] += d0; cb[2 * j + 1] += d1;
          const uint32_t dp = pack_h2<BF16>(d0, d1);
          g2p[2 * j + h] = dp;
          if constexpr (kStageDg2) {
            const uint32_t wa = g1_word(c, rb + 8 * h);
            if constexpr (ACT != DIB_ACT_LINEAR) {
              float x0, x1;
              unpack_h2<BF16>(ld_shared_b32(wa), x0, x1);
              g1m[j >> 3] |= (x0 > 0.f ? 1u : 0u) << (4 * (j & 7) + 2 * h) | (x1 > 0.f ? 2u : 0u) << (4 * (j & 7) + 2 * h);
            }
            st_shared_b32(wa, dp);
          } else if (row_lo + 8 * h < a.M) *reinterpret_cast<uint32_t*>(a.dg2 + (row_lo + 8 * h) * a.lddg + c) = dp;
        }
      }
      quad_col_sums<kF2N / 8>(cb, s_col[warp], lane);
      if constexpr (kStageDg2) {
        fence_proxy_async_smem();
        named_bar_sync(2 + wg, 128);
        store_panels(&mapDg2, tile, 0, kF2N / 64, 0);
      }
      named_bar_sync(1, kConsumers);
#pragma unroll
      for (int w = 0; w < kConsumers / 32; ++w) acc_dbh += s_col[w][tid];
      named_bar_sync(1, kConsumers);
    }
    if (bwd) {
      // ---------------- D1, e2 per 128-column chunk: dg1 = (dg2 W1^T) act'(g1) -> over the chunk's g1 in the shared tile (each
      // thread overwrites the words it reads) -> HBM, and packed into dg1p (A of D0); column sums -> dbpart row of the tile
      uint32_t dg1p[64];
      float acc2[64];
#pragma unroll
      for (int cc = 0; cc < kF2N / kF2BtN; ++cc) {
#pragma unroll
        for (int i = 0; i < 64; ++i) acc2[i] = 0.f;
        mainloop_rs(acc2, g2p);
        // the store group that last read the tile (kStageDg2: dg2's; else g1's) is done before dg1 goes over panels 0-1
        if (cc == 0) stores_drained(std::integral_constant<int, 0>());
#pragma unroll
        for (int j = 0; j < kF2BtN / 8; ++j) {
          const int c = kF2BtN * cc + 8 * j + 2 * q;
          float cs[2] = {0.f, 0.f};
#pragma unroll
          for (int h = 0; h < 2; ++h) {
            const uint32_t wa = g1_word(c, rb + 8 * h);
            float f0, f1;                                  // act'(g1): the floats dib_act_grad returns, as factors
            if constexpr (kStageDg2) {
              const int jj = kF2BtN / 8 * cc + j, b = 4 * (jj & 7) + 2 * h;
              const float off = ACT == DIB_ACT_LEAKY_RELU ? a.alpha : 0.f;
              f0 = ACT == DIB_ACT_LINEAR || (g1m[jj >> 3] >> b & 1u) ? 1.f : off;
              f1 = ACT == DIB_ACT_LINEAR || (g1m[jj >> 3] >> (b + 1) & 1u) ? 1.f : off;
            } else {
              float x0, x1;
              unpack_h2<BF16>(ld_shared_b32(wa), x0, x1);
              f0 = dib_act_grad(ACT, x0, a.alpha); f1 = dib_act_grad(ACT, x1, a.alpha);
            }
            const float v0 = acc2[4 * j + 2 * h] * f0;
            const float v1 = acc2[4 * j + 2 * h + 1] * f1;
            const uint32_t p = pack_h2<BF16>(v0, v1);
            dg1p[2 * (kF2BtN / 8 * cc + j) + h] = p;
            st_shared_b32(wa, p);
            if (row_lo + 8 * h < a.M) { cs[0] += v0; cs[1] += v1; }   // rows outside the matrix add nothing
          }
          cs[0] = quad_col_sum(cs[0]); cs[1] = quad_col_sum(cs[1]);
          if (lane < 4) { s_col[warp][c] = cs[0]; s_col[warp][c + 1] = cs[1]; }
        }
        fence_proxy_async_smem();
        named_bar_sync(2 + wg, 128);
        store_panels(&mapDg1, tile, 2 * cc, kF2BtN / 64, kF2BtN * cc);
      }
      named_bar_sync(1, kConsumers);
      {
        float sum = 0.f;
#pragma unroll
        for (int w = 0; w < kConsumers / 32; ++w) sum += s_col[w][tid];
        a.dbpart[(long long)tile * kF2N + tid] = sum;
      }
      named_bar_sync(1, kConsumers);
      // ---------------- D0, e3: d emb = dg1 W0^T per 128-column chunk -> two 64-column panels of the warpgroup's rows of the
      // g1 tile (chunks alternate between panels 0-1 and 2-3, as the dg1 stores did, so a chunk waits only for the store
      // group before last) -> TMA store
      for (int c0 = 0, cc = 0; c0 < a.demb_cols; c0 += kF2BtN, ++cc) {
#pragma unroll
        for (int i = 0; i < 64; ++i) acc2[i] = 0.f;
        mainloop_rs(acc2, dg1p);
        stores_drained(std::integral_constant<int, 1>());
        const int tc = (cc & 1) * kF2BtN;                 // shared-tile columns of this chunk
#pragma unroll
        for (int j = 0; j < kF2BtN / 8; ++j) {
#pragma unroll
          for (int h = 0; h < 2; ++h)
            st_shared_b32(g1_word(tc + 8 * j + 2 * q, rb + 8 * h), pack_h2<BF16>(acc2[4 * j + 2 * h], acc2[4 * j + 2 * h + 1]));
        }
        fence_proxy_async_smem();
        named_bar_sync(2 + wg, 128);
        store_panels(&mapDemb, tile, tc / 64, min(kF2BtN, a.demb_cols - c0) / 64, c0);
      }
    }
  }
  if ((tid & 127) == 0) bulk_wait_all();
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

// WEIGHTED: row i's loss and d loss / d z carry its sample weight wts[i]
template <int KPT, int OUT, int ROWS, bool BF16, bool WEIGHTED>   // hidden units per lane (K / 32); bound of the output width; rows in flight per warp
__global__ void __launch_bounds__(kHeadWarps * 32)
dib_int16_head_kernel(const uint16_t* __restrict__ g, int ldg, int K, const float* __restrict__ Wc, const float* __restrict__ bc,
                      int out_dim, int out_act, int hid_act, float alpha, int loss, const float* __restrict__ y, long long n,
                      float inv_batch, float gscale, uint16_t* __restrict__ dg, int lddg, float* __restrict__ user_pred,
                      float* __restrict__ wpart, int wpart_stride, float* __restrict__ loss_part, float* __restrict__ acc_part,
                      const float* __restrict__ wts) {
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
      float wr = 1.f, ib = inv_batch;
      if constexpr (WEIGHTED) { wr = wts[row]; ib *= wr; }
      if (y) {
        float l = 0.f, acc = 0.f;
        const float inv_out = 1.f / (float)out_dim;
        if (loss == DIB_LOSS_SPARSE_CE_LOGITS) {
          const int label = dib_sparse_label(y[row], out_dim);     // < 0: NaN loss and gradient (an invalid label)
          float m = z[0], zl = __int_as_float(0x7fc00000), se = 0.f; int am = 0;
#pragma unroll
          for (int o = 1; o < OUT; ++o) if (o < out_dim && z[o] > m) { m = z[o]; am = o; }
#pragma unroll
          for (int o = 0; o < OUT; ++o) if (o < out_dim) { se += expf(z[o] - m); if (o == label) zl = z[o]; }
          l = m + logf(se) - zl;
          if constexpr (WEIGHTED) l *= wr;
          acc = (float)am == y[row] ? 1.f : 0.f;
#pragma unroll
          for (int o = 0; o < OUT; ++o)
            if (o < out_dim) dz[o] = label < 0 ? __int_as_float(0x7fc00000) : expf(z[o] - m) / se - (o == label ? 1.f : 0.f);
        } else {
#pragma unroll
          for (int o = 0; o < OUT; ++o) if (o < out_dim) {
            dz[o] = dib_loss_add_t<WEIGHTED>(loss, z[o], y[row * out_dim + o], wr, l, acc) * inv_out;
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
        for (int o = 0; o < OUT; ++o) { dz[o] *= ib * dib_act_grad(out_act, z[o], alpha); db[o] += dz[o]; }
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
template <bool BF16, bool WEIGHTED>       // WEIGHTED: as the generic kernel
__global__ void __launch_bounds__(kHeadWarps * 32)
dib_int16_head1_kernel(const uint16_t* __restrict__ g, int ldg, int K, const float* __restrict__ Wc, const float* __restrict__ bc,
                       int out_act, int hid_act, float alpha, int loss, const float* __restrict__ y, long long n,
                       float inv_batch, float gscale, uint16_t* __restrict__ dg, int lddg, float* __restrict__ user_pred,
                       float* __restrict__ wpart, int wpart_stride, float* __restrict__ loss_part, float* __restrict__ acc_part,
                       const float* __restrict__ wts) {
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
    float dz = 0.f, ib = inv_batch;
    if (live && y) {
      const float t = y[mrow];
      float wr = 1.f;
      if constexpr (WEIGHTED) { wr = wts[mrow]; ib *= wr; }
      float l = -0.f, acc = -0.f;
      if (loss == DIB_LOSS_SPARSE_CE_LOGITS) {     // one class: the softmax is constant; an invalid label gives NaN
        l = dz = dib_sparse_label(t, 1) < 0 ? __int_as_float(0x7fc00000) : 0.f;
        acc = t == 0.f ? 1.f : 0.f;
      }
      else dz = dib_loss_add_t<WEIGHTED>(loss, z, t, wr, l, acc);
      if (lane < ROWS) { lsum += l; asum += acc; }
    }
    if (user_pred && live && lane < ROWS) user_pred[mrow] = z;
    if (train) {
      dz = live ? dz * ib * dib_act_grad(out_act, z, alpha) : 0.f;
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
    cudaError_t e = cudaFuncSetAttribute(dib_int16_gemm_kernel<MODE, BF16>, cudaFuncAttributeMaxDynamicSharedMemorySize, kGemmSmem);
    if (e != cudaSuccess) return e;
    attr = true;
  }
  dib_int16_gemm_kernel<MODE, BF16><<<(unsigned)(ntile < cap ? ntile : cap), kGemmThreads, kGemmSmem, st>>>(mA, mB, a, mA2, mB2, a2);
  dib_note_launch();
  return cudaGetLastError();
}

struct ConvSegs { const float* src[8]; uint16_t* dst[8]; long long first[9]; int nseg; };
template <bool BF16>
__global__ void dib_f32_to_16_segs_kernel(const ConvSegs A) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= A.first[A.nseg]) return;
  int k = 0;
#pragma unroll
  for (int q = 1; q < 8; ++q) if (q < A.nseg && i >= A.first[q]) k = q;
  // saturating like every activation operand: a weight beyond fp16's 65 504 converts to +-65 504, not inf
  A.dst[k][i - A.first[k]] = (uint16_t)(pack_h2<BF16>(A.src[k][i - A.first[k]], 0.f) & 0xffffu);
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

// g_out[M x N] = act(g_in[M x K] W16[K x N] + bias)
cudaError_t dib_int16_fwd(const void* g_in, int ld_in, const void* w16, const float* bias, void* g_out, int ld_out, int M,
                          int K, int N, int act, float alpha, int bf16, cudaStream_t st) {
  if (!encode_fn3()) return cudaErrorNotSupported;
  CUtensorMap mA, mB;
  if (!map_k(&mA, g_in, K, M, ld_in, kBM) || !map_mn(&mB, w16, N, K, N, kBN / 64))
    return cudaErrorInvalidValue;
  Int16Args a{};
  a.out16 = static_cast<uint16_t*>(g_out); a.ldc = ld_out; a.bias = bias; a.M = M; a.T = K; a.C = N; a.act = act; a.alpha = alpha;
  a.out_scale = 1.f; a.nsplit = 1;
  const long long nt = (long long)DIB_CEIL_DIV(M, kBM) * DIB_CEIL_DIV(N, kBN);
  return bf16 ? launch16<DIB_GEMM_FWD, true>(mA, mB, a, mA, mB, Int16Args{}, nt, st)
              : launch16<DIB_GEMM_FWD, false>(mA, mB, a, mA, mB, Int16Args{}, nt, st);
}

// dz_in[M x K] = (dz[M x N] W16[K x N]^T) * act'(g_in[M x K])      (g_in may be null: no activation, e.g. d_emb)
cudaError_t dib_int16_dgrad(const void* dz, int ld_dz, const void* w16, const void* g_in, int ld_g, void* dz_in, int ld_out,
                            int M, int K, int N, int act, float alpha, float* colsum_part, int bf16, cudaStream_t st) {
  if (!encode_fn3()) return cudaErrorNotSupported;
  CUtensorMap mA, mB;
  if (!map_k(&mA, dz, N, M, ld_dz, kBM) || !map_k(&mB, w16, N, K, N, kBN))
    return cudaErrorInvalidValue;
  Int16Args a{};
  a.out16 = static_cast<uint16_t*>(dz_in); a.ldc = ld_out; a.X = static_cast<const uint16_t*>(g_in); a.ldx = ld_g;
  a.M = M; a.T = N; a.C = K; a.act = act; a.alpha = alpha; a.out_scale = 1.f; a.nsplit = 1; a.dbias = colsum_part;
  const long long nt = (long long)DIB_CEIL_DIV(M, kBM) * DIB_CEIL_DIV(K, kBN);
  return bf16 ? launch16<DIB_GEMM_DGRAD, true>(mA, mB, a, mA, mB, Int16Args{}, nt, st)
              : launch16<DIB_GEMM_DGRAD, false>(mA, mB, a, mA, mB, Int16Args{}, nt, st);
}

// dW (fp32 split partials, * out_scale) = g_in^T dz of one or two layers.  Two layers' tiles fill a wave of CTAs that one
// layer's do not.  The bias gradients come from the kernel that produces dz (dgrad epilogue / output head), not from here.
cudaError_t dib_int16_wgrad(const DibInt16Wgrad* layers, int count, int M, long long split_stride, float out_scale, int bf16,
                            cudaStream_t st) {
  if (count < 1 || count > 2) return cudaErrorInvalidValue;
  if (!encode_fn3()) return cudaErrorNotSupported;
  CUtensorMap mA[2], mB[2];
  Int16Args a[2] = {};              // a[1].nsplit == 0: no second problem
  long long nt = 0;
  for (int q = 0; q < count; ++q) {
    const DibInt16Wgrad& l = layers[q];
    if (!map_mn(&mA[q], l.g_in, l.K, M, l.K, kBM / 64) || !map_mn(&mB[q], l.dz, l.N, M, l.N, kBN / 64))
      return cudaErrorInvalidValue;
    a[q].out32 = l.dW_part; a[q].ldc = l.N; a[q].M = M; a[q].C = l.N; a[q].R = l.K; a[q].out_scale = out_scale;
    a[q].nsplit = l.nsplit; a[q].rows_per_split = l.rows_per_split; a[q].split_stride = split_stride;
    nt += (long long)DIB_CEIL_DIV(l.K, kBM) * DIB_CEIL_DIV(l.N, kBN) * l.nsplit;
  }
  if (count == 1) { mA[1] = mA[0]; mB[1] = mB[0]; }
  return bf16 ? launch16<DIB_GEMM_WGRAD, true>(mA[0], mB[0], a[0], mA[1], mB[1], a[1], nt, st)
              : launch16<DIB_GEMM_WGRAD, false>(mA[0], mB[0], a[0], mA[1], mB[1], a[1], nt, st);
}

// whole kBK-column k-blocks of the fan-in and whole kBN-column tiles of the fan-out
bool dib_int16_gemm_ok(int K, int N) { return K >= kBK && K % kBK == 0 && N >= kBN && N % kBN == 0; }

bool dib_int16_fwd2_ok(int K0, int N1, int N2, int out_dim) {
  return dib_int16_gemm_ok(K0, N1) && N1 == kF2N && N2 == kF2N && out_dim == 1;
}

// g1 = act(g_in W0 + b0) -> HBM;  g2 = act(g1 W1 + b1) (on chip);  logit = g2 . wout + bout;  compiled loss / metric;
// training (dg2 != null): dg2, per-CTA partials of the output layer's gradients and of the last hidden layer's bias gradient;
// and with dg1 != null the dgrad of the second layer, dg1 = (dg2 W1^T) act'(g1) with its per-tile column sums in dbpart
// [ceil(M/128)][256] (as dib_int16_dgrad), and with demb != null (g_in has no activation: the embedding) also
// demb [M x K0] = dg1 W0^T.  *nblocks = CTAs launched = rows of wpart / loss_part / acc_part written.
cudaError_t dib_int16_fwd2_head(const void* g_in, int ld_in, int K0, const void* w16_0, const float* b0, const void* w16_1, const float* b1,
                                void* g1, const float* wout, const float* bout, int act, int out_act, float alpha, int loss, const float* y,
                                int M, float inv_batch, float gscale, void* dg2, void* dg1, float* dbpart, void* demb, float* user_pred,
                                float* wpart, int wpart_stride, float* loss_part, float* acc_part, int* nblocks, const float* weights,
                                int bf16, cudaStream_t st) {
  if (!encode_fn3()) return cudaErrorNotSupported;
  if ((dg1 && (!dg2 || !dbpart)) || (demb && !dg1)) return cudaErrorInvalidValue;
  CUtensorMap mA, mW0, mW1;
  if (!map_k(&mA, g_in, K0, M, ld_in, kBM) || !map_mn(&mW0, w16_0, kF2N, K0, kF2N, kF2N / 64) || !map_mn(&mW1, w16_1, kF2N, kF2N, kF2N, kF2N / 64))
    return cudaErrorInvalidValue;
  // the store maps of g1, dg1, dg2 and d emb (box 64 x 64: one panel of a warpgroup's rows); backward stages: W1 and W0 K-major
  // (box 64 x 128, as dib_int16_dgrad reads them)
  CUtensorMap mG1, mW1t = mA, mW0t = mA, mDg1 = mA, mDg2 = mA, mDemb = mA;
  if (!map_k(&mG1, g1, kF2N, M, kF2N, 64)) return cudaErrorInvalidValue;
  if (dg2 && !map_k(&mDg2, dg2, kF2N, M, kF2N, 64)) return cudaErrorInvalidValue;   // relu / leaky relu / linear
  if (dg1 && (!map_k(&mW1t, w16_1, kF2N, kF2N, kF2N, kF2BtN) || !map_k(&mDg1, dg1, kF2N, M, kF2N, 64))) return cudaErrorInvalidValue;
  if (demb && (!map_k(&mW0t, w16_0, kF2N, K0, kF2N, kF2BtN) || !map_k(&mDemb, demb, K0, M, K0, 64))) return cudaErrorInvalidValue;
  Fwd2Args a{};
  a.b0 = b0; a.b1 = b1; a.wout = wout; a.bout = bout;
  a.dg2 = static_cast<uint16_t*>(dg2); a.lddg = kF2N; a.y = y; a.user_pred = user_pred; a.wts = weights; a.wpart = wpart; a.wpart_stride = wpart_stride;
  a.bwd = dg1 != nullptr; a.dbpart = dbpart; a.demb_cols = demb ? K0 : 0;
  a.loss_part = loss_part; a.acc_part = acc_part; a.M = M; a.nk0 = K0 / kBK; a.act = act; a.out_act = out_act; a.loss = loss;
  a.alpha = alpha; a.inv_batch = inv_batch; a.gscale = gscale;
  const int tiles = DIB_CEIL_DIV(M, kBM);
  const int grid = tiles < num_sms16() ? tiles : num_sms16();
  *nblocks = grid;
  if (grid <= 0) return cudaSuccess;
  cudaError_t e = cudaErrorInvalidValue;
#define DIB_F2_LAUNCH(BF, ACT, W)                                                                                                    \
  do {                                                                                                                               \
    static bool attr = false;                                                                                                        \
    e = attr ? cudaSuccess : cudaFuncSetAttribute(dib_int16_fwd2_kernel<BF, ACT, W>, cudaFuncAttributeMaxDynamicSharedMemorySize, kF2Smem); \
    if (e != cudaSuccess) return e;                                                                                                  \
    attr = true;                                                                                                                     \
    dib_int16_fwd2_kernel<BF, ACT, W><<<grid, kF2Threads, kF2Smem, st>>>(mA, mW0, mW1, mW1t, mW0t, mDemb, mG1, mDg1, mDg2, a);      \
  } while (0)
#define DIB_F2_BF(ACT, W) do { if (bf16) DIB_F2_LAUNCH(true, ACT, W); else DIB_F2_LAUNCH(false, ACT, W); } while (0)
#define DIB_F2_ACT(ACT) do { if (weights) DIB_F2_BF(ACT, true); else DIB_F2_BF(ACT, false); } while (0)
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
#undef DIB_F2_BF
#undef DIB_F2_LAUNCH
  dib_note_launch();
  return cudaGetLastError();
}

int dib_int16_head_blocks(int num_sms) { return num_sms * 2; }

// the kernels are launched with 8 hidden units per lane: K = 256
bool dib_int16_head_ok(int K, int out_dim, bool head1) {
  return K == 8 * 32 && out_dim >= 1 && out_dim <= kHeadMaxOut && (!head1 || out_dim == 1);
}

cudaError_t dib_int16_head(const void* g, int ldg, int K, const float* Wc, const float* bc, int out_dim, int out_act, int hid_act,
                           float alpha, int loss, const float* y, long long n, float inv_batch, float gscale, void* dg, int lddg,
                           float* user_pred, float* wpart, int wpart_stride, float* loss_part, float* acc_part, int nblocks,
                           bool head1, const float* weights, int bf16, cudaStream_t st) {
  if (!dib_int16_head_ok(K, out_dim, head1)) return cudaErrorInvalidValue;
#define DIB_HEAD_T(OUT, BF, W)                                                                                          \
  dib_int16_head_kernel<8, OUT, (OUT <= 2 ? 4 : 1), BF, W><<<nblocks, kHeadWarps * 32, 0, st>>>(static_cast<const uint16_t*>(g), ldg, K, Wc, bc, out_dim,  \
      out_act, hid_act, alpha, loss, y, n, inv_batch, gscale, static_cast<uint16_t*>(dg), lddg, user_pred, wpart, wpart_stride, \
      loss_part, acc_part, weights)
#define DIB_HEAD_W(OUT, W) do { if (bf16) DIB_HEAD_T(OUT, true, W); else DIB_HEAD_T(OUT, false, W); } while (0)
#define DIB_HEAD(OUT) do { if (weights) DIB_HEAD_W(OUT, true); else DIB_HEAD_W(OUT, false); } while (0)
#define DIB_HEAD1(BF, W)                                                                                                \
  dib_int16_head1_kernel<BF, W><<<nblocks, kHeadWarps * 32, 0, st>>>(static_cast<const uint16_t*>(g), ldg, K, Wc, bc, out_act, hid_act,  \
      alpha, loss, y, n, inv_batch, gscale, static_cast<uint16_t*>(dg), lddg, user_pred, wpart, wpart_stride, loss_part, acc_part, weights)
  if (head1) {
    if (bf16) { if (weights) DIB_HEAD1(true, true); else DIB_HEAD1(true, false); }
    else { if (weights) DIB_HEAD1(false, true); else DIB_HEAD1(false, false); }
  } else if (out_dim == 1) DIB_HEAD(1);
  else if (out_dim == 2) DIB_HEAD(2);
  else if (out_dim <= 4) DIB_HEAD(4);
  else if (out_dim <= 8) DIB_HEAD(8);
  else DIB_HEAD(16);
#undef DIB_HEAD1
#undef DIB_HEAD
#undef DIB_HEAD_W
#undef DIB_HEAD_T
  dib_note_launch();
  return cudaGetLastError();
}
