// dib_gemm_tc.cu -- grouped TF32 tensor-core GEMMs (wgmma .tf32, fp32 accumulators in registers, mbarrier pipeline,
// warp-specialised) with the same fused epilogues and the same problem descriptors as the fp32 SIMT path
// (dib_gemm_simt.cu).  TF32 reads the existing fp32 activation / weight buffers directly: the MMAs consume the 32-bit
// containers, so no conversion pass and no second copy of the data exist.
//
// Canonical form Out[R x C] = sum_t Aop[R x T] * Bop[T x C]; operand majors per mode
//   FWD    A = h[M x K]   K-major | B = W[K x N]        MN-major      (reduction over fan-in)
//   DGRAD  A = dz[M x N]  K-major | B = W[K x N] as [k][n] K-major    (reduction over fan-out)
//   WGRAD  A = h[m][k]   MN-major | B = dz[m][n]        MN-major      (reduction over a batch slice)
// wgmma reads tf32 operands K-major only: K-major operands arrive by TMA (SWIZZLE_128B), MN-major operands are transposed
// by the producer warpgroup on their way from global into the same swizzled K-major layout.
// CTA tile 128 x BN (BN = 64 | 128), K step 32 fp32 (= one 128-byte swizzle span) per pipeline stage.
// Warps: 0..7 two consumer warpgroups (MMAs + epilogue of rows [64 g, 64 g + 64)) | 8..11 producer warpgroup.
#include <cuda.h>

#include <cstdio>
#include <cstring>

#include "dib_common.cuh"
#include "dib_kernels.h"
#include "dib_sm90.cuh"

namespace {

using namespace sm90;

constexpr int kBM = 128, kBK = 32, kStages = 4;
constexpr int kABytes = kBM * 128;   // 128 rows x 128 B (32 fp32 of K per row)
constexpr int kConsumers = 256, kThreads = kConsumers + 128;

template <int BN>
struct SmemLayout {
  static constexpr int kBBytes = BN * 128;
  static constexpr int kStageBytes = kABytes + kBBytes;
  static constexpr int kBarOff = kStages * kStageBytes;          // full[S], empty[S]
  static constexpr int kTotal = kBarOff + 128 + 1024;            // + alignment slack
};

__device__ __forceinline__ void st_shared_f32(uint32_t addr, float v) {
  asm volatile("st.shared.f32 [%0], %1;" ::"r"(addr), "f"(v) : "memory");
}

// Producer warpgroup: a [32 k][ROWS mn] fp32 tile whose mn is contiguous in global memory (element (k, mn) at
// src[k * ld + mn]) -> the K-major swizzled stage tile [ROWS][128 B]: row mn, 16-byte chunk (k / 4) ^ (mn % 8), word k % 4.
// Lane = k, so the 32 lanes of a store hit 32 different banks.  Rows k >= k_end and columns mn >= mn_end read as zero.
// sum: add the values to this thread's running column sums (column 4 (pw + 4 i) + e at index 4 i + e).
template <int ROWS>
__device__ __forceinline__ void load_transposed(uint32_t dst, const float* src, long long ld, int k0, int k_end, int mn0, int mn_end,
                                                int pw, int lane, bool sum, float (&colsum)[ROWS / 4]) {
  constexpr int NV = ROWS / 16;                   // float4 per thread: ROWS / 4 groups of 4 columns over 4 producer warps
  const int k = k0 + lane;
  const float* row = src + (long long)k * ld;
  float4 v[NV];
#pragma unroll
  for (int i = 0; i < NV; ++i) {
    const int mn = mn0 + 4 * (pw + 4 * i);
    v[i] = (k < k_end && mn < mn_end) ? *reinterpret_cast<const float4*>(row + mn) : make_float4(0.f, 0.f, 0.f, 0.f);
  }
#pragma unroll
  for (int i = 0; i < NV; ++i) {
    const float e[4] = {v[i].x, v[i].y, v[i].z, v[i].w};
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int r = 4 * (pw + 4 * i) + j;
      st_shared_f32(dst + r * 128 + (((lane >> 2) ^ (r & 7)) << 4) + (lane & 3) * 4, e[j]);
      if (sum) colsum[4 * i + j] += e[j];
    }
  }
}

template <int MODE, int BN>
__global__ void __launch_bounds__(kThreads, 1)
dib_gemm_tc_kernel(const __grid_constant__ CUtensorMap mapA, const __grid_constant__ CUtensorMap mapB,
                   const DibGemmProblem* __restrict__ probs, const float* __restrict__ baseA, const float* __restrict__ baseB,
                   const float* __restrict__ baseP, float* __restrict__ baseC, float* baseX, int M, int nsplit,
                   int rows_per_split, long long split_stride, float alpha, int round_out) {
  using L = SmemLayout<BN>;
  constexpr bool A_MN = (MODE == DIB_GEMM_WGRAD), B_MN = (MODE != DIB_GEMM_DGRAD);
  extern __shared__ uint8_t smem_raw[];
  const uint32_t smem_base = (smem_u32(smem_raw) + 1023u) & ~1023u;
  const uint32_t bar_base = smem_base + L::kBarOff;
  auto full_bar = [&](int s) { return bar_base + 8u * s; };
  auto empty_bar = [&](int s) { return bar_base + 8u * (kStages + s); };

  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  int prob, split = 0, r0, c0;
  if constexpr (MODE == DIB_GEMM_WGRAD) {
    prob = blockIdx.z / nsplit; split = blockIdx.z % nsplit;
    c0 = blockIdx.x * BN; r0 = blockIdx.y * kBM;
  } else {
    prob = blockIdx.z; r0 = blockIdx.x * kBM; c0 = blockIdx.y * BN;
  }
  const DibGemmProblem p = probs[prob];
  const int R = (MODE == DIB_GEMM_WGRAD) ? p.R : M;
  const int C = p.C;
  int t_begin = 0, t_end = p.T;
  if constexpr (MODE == DIB_GEMM_WGRAD) {
    t_begin = split * rows_per_split;
    t_end = min(M, t_begin + rows_per_split);
  }
  if (r0 >= R || c0 >= C) return;                       // uniform per CTA
  const int ntiles = t_end > t_begin ? DIB_CEIL_DIV(t_end - t_begin, kBK) : 0;
  const bool do_db = (MODE == DIB_GEMM_WGRAD) && (blockIdx.y == 0) && (p.x_off >= 0);
  // arrivals that complete a stage: the TMA issuer's expect_tx, and every producer thread that stored a transposed operand
  constexpr uint32_t kTmaBytes = (A_MN ? 0 : kABytes) + (B_MN ? 0 : L::kBBytes);
  constexpr uint32_t kFullCount = (kTmaBytes ? 1 : 0) + ((A_MN || B_MN) ? 128 : 0);

  if (tid == 0) {
    for (int s = 0; s < kStages; ++s) {
      mbar_init(full_bar(s), kFullCount);
      mbar_init(empty_bar(s), kConsumers / 32);          // every consumer warp releases the stage
    }
    fence_barrier_init();
  }
  __syncthreads();

  if (warp >= kConsumers / 32) {
    // ============================================================== producer warpgroup
    const int pt = tid - kConsumers, pw = pt >> 5;
    if (pt == 0) {
      if (kTmaBytes) { tma_prefetch_desc(&mapA); tma_prefetch_desc(&mapB); }
    }
    float cs[BN / 4], cs_a[kBM / 4];                      // bias gradient (WGRAD): column sums of this thread's dz values
#pragma unroll
    for (int i = 0; i < BN / 4; ++i) cs[i] = 0.f;
    for (int it = 0; it < ntiles; ++it) {
      const int s = it % kStages, ph = (it / kStages) & 1;
      mbar_wait(empty_bar(s), ph ^ 1);
      const uint32_t a_dst = smem_base + s * L::kStageBytes, b_dst = a_dst + kABytes;
      const int t0 = t_begin + it * kBK;
      if (kTmaBytes && pt == 0) {
        mbar_expect_tx(full_bar(s), kTmaBytes);
        if constexpr (!A_MN) tma_load_3d(a_dst, &mapA, full_bar(s), t0, r0, prob);
        if constexpr (!B_MN) tma_load_3d(b_dst, &mapB, full_bar(s), t0, c0, prob);
      }
      if constexpr (A_MN || B_MN) {
        if constexpr (A_MN) load_transposed<kBM>(a_dst, baseA + p.a_off, p.lda, t0, t_end, r0, p.lda, pw, lane, false, cs_a);
        if constexpr (B_MN) load_transposed<BN>(b_dst, baseB + p.b_off, p.ldb, t0, t_end, c0, p.ldb, pw, lane, do_db, cs);
        fence_proxy_async_smem();
        mbar_arrive(full_bar(s));
      }
    }
    if (do_db) {
      // column 4 (pw + 4 i) + e of the tile: this warp's 32 k rows per stage summed over the stages, then over the lanes (fixed order)
#pragma unroll
      for (int i = 0; i < BN / 4; ++i) cs[i] = dib_warp_sum(cs[i]);
      if (lane == 0) {
        float* db = baseX + p.x_off + (long long)split * split_stride;
#pragma unroll
        for (int i = 0; i < BN / 16; ++i)
#pragma unroll
          for (int e = 0; e < 4; ++e) {
            const int c = c0 + 4 * (pw + 4 * i) + e;
            if (c < C) db[c] = cs[4 * i + e];
          }
      }
    }
  } else {
    // ============================================================== consumer warpgroups: MMAs + epilogue
    const int wg = tid >> 7, q = lane & 3;
    const int rb = 64 * wg + 16 * (warp & 3) + (lane >> 2);
    float acc[BN / 2];
#pragma unroll
    for (int i = 0; i < BN / 2; ++i) acc[i] = 0.f;
    if (ntiles > 0) {
      int prev = 0;
      for (int it = 0; it < ntiles; ++it) {
        const int s = it % kStages, ph = (it / kStages) & 1;
        mbar_wait(full_bar(s), ph);
        const uint32_t a_addr = smem_base + s * L::kStageBytes + wg * 64 * 128, b_addr = smem_base + s * L::kStageBytes + kABytes;
        wgmma_fence();
#pragma unroll
        for (int kk = 0; kk < kBK / 8; ++kk) {          // wgmma K = 8 for tf32 (32 bytes)
          const uint64_t da = gmma_desc(a_addr + kk * 32, 16, 1024), db = gmma_desc(b_addr + kk * 32, 16, 1024);
          if constexpr (BN == 128) wgmma_tf32_m64n128k8(acc, da, db, (it > 0 || kk > 0) ? 1u : 0u);
          else wgmma_tf32_m64n64k8(acc, da, db, (it > 0 || kk > 0) ? 1u : 0u);
        }
        wgmma_commit();
        wgmma_wait<1>();
        if (it > 0 && lane == 0) mbar_arrive(empty_bar(prev));
        prev = s;
      }
      wgmma_wait<0>();
      if (lane == 0) mbar_arrive(empty_bar(prev));
      wgmma_fence_regs(acc);
    }
    float* __restrict__ Out = baseC + p.c_off + (MODE == DIB_GEMM_WGRAD ? (long long)split * split_stride : 0ll);
#pragma unroll
    for (int j = 0; j < BN / 8; ++j) {
      const int c = c0 + 8 * j + 2 * q;
      if (c >= C) continue;
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int r = r0 + rb + 8 * h;
        if (r >= R) continue;
        float2 o = make_float2(acc[4 * j + 2 * h], acc[4 * j + 2 * h + 1]);
        if constexpr (MODE == DIB_GEMM_FWD) {
          const float2 b = *reinterpret_cast<const float2*>(baseP + p.x_off + c);
          o.x = dib_maybe_round(dib_act(p.act, o.x + b.x, alpha), round_out);
          o.y = dib_maybe_round(dib_act(p.act, o.y + b.y, alpha), round_out);
        } else if constexpr (MODE == DIB_GEMM_DGRAD) {
          if (p.act != DIB_ACT_LINEAR) {
            const float2 x = *reinterpret_cast<const float2*>(baseX + p.x_off + (long long)r * p.ldx + c);
            o.x *= dib_act_grad(p.act, x.x, alpha);
            o.y *= dib_act_grad(p.act, x.y, alpha);
          }
          o.x = dib_maybe_round(o.x, round_out);
          o.y = dib_maybe_round(o.y, round_out);
        }
        *reinterpret_cast<float2*>(Out + (long long)r * p.ldc + c) = o;
      }
    }
  }
}

// ------------------------------------------------------------------------------------------------ host side
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                  const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                  CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

EncodeTiledFn encode_fn() {
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

// K-major operand: matrix [rows x ld] fp32, feature stride fs floats -> 3D map (col, row, feature), box 32 x brows x 1
bool make_map_kmajor(CUtensorMap* m, const float* base, long long cols, long long rows, long long ld, long long fs,
                     int nfeat, int box_rows) {
  cuuint64_t dims[3] = {(cuuint64_t)cols, (cuuint64_t)rows, (cuuint64_t)nfeat};
  cuuint64_t strides[2] = {(cuuint64_t)ld * 4, (cuuint64_t)(nfeat > 1 ? fs : ld * rows) * 4};
  cuuint32_t box[3] = {32, (cuuint32_t)box_rows, 1};
  cuuint32_t es[3] = {1, 1, 1};
  return encode_fn()(m, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 3, const_cast<float*>(base), dims, strides, box, es,
                     CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                     CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) == CUDA_SUCCESS;
}

template <int MODE, int BN>
cudaError_t launch_tc(const DibGemmLaunch& L, const CUtensorMap& mapA, const CUtensorMap& mapB, cudaStream_t st) {
  using SL = SmemLayout<BN>;
  static bool attr_set = false;
  auto kern = dib_gemm_tc_kernel<MODE, BN>;
  if (!attr_set) {
    cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, SL::kTotal);
    if (e != cudaSuccess) return e;
    attr_set = true;
  }
  dim3 grid;
  if (MODE == DIB_GEMM_WGRAD)
    grid = dim3(DIB_CEIL_DIV(L.maxC, BN), DIB_CEIL_DIV(L.maxR, kBM), L.nprob * L.nsplit);
  else
    grid = dim3(DIB_CEIL_DIV(L.M, kBM), DIB_CEIL_DIV(L.maxC, BN), L.nprob);
  if (grid.x == 0 || grid.y == 0 || grid.z == 0) return cudaSuccess;
  kern<<<grid, kThreads, SL::kTotal, st>>>(mapA, mapB, L.probs, L.baseA, L.baseB, L.baseBias ? L.baseBias : L.baseB, L.baseC,
                                           L.baseX, L.M, L.nsplit, L.rows_per_split, L.split_stride, L.alpha, L.round_out);
  dib_note_launch();
  return cudaGetLastError();
}

}  // namespace

// Can this group of problems (host copies) run on the tensor-core kernel?  See the operand-major table above.
bool dib_gemm_tc_eligible(int mode, const DibGemmProblem* hp, int nprob, const float* params_base_hint) {
  (void)params_base_hint;
  if (!encode_fn() || nprob < 1) return false;
  const DibGemmProblem& p0 = hp[0];
  const long long sa = nprob > 1 ? hp[1].a_off - hp[0].a_off : 0, sb = nprob > 1 ? hp[1].b_off - hp[0].b_off : 0;
  for (int i = 0; i < nprob; ++i) {
    const DibGemmProblem& p = hp[i];
    if (p.T != p0.T || p.C != p0.C || p.R != p0.R || p.lda != p0.lda || p.ldb != p0.ldb || p.ldc != p0.ldc) return false;
    if (p.a_off != p0.a_off + i * sa || p.b_off != p0.b_off + i * sb) return false;
    if ((p.a_off & 3) || (p.b_off & 3) || (p.c_off & 3) || (p.x_off & 3)) return false;
  }
  if ((sa & 3) || (sb & 3) || sa < 0 || sb < 0) return false;
  if (p0.C % 64) return false;
  if (p0.lda < 32 || p0.ldb < 32 || (p0.ldc & 3)) return false;
  switch (mode) {
    case DIB_GEMM_FWD:   return p0.T >= 32 && (p0.ldb % 32) == 0;               // W panels of 32 along N
    case DIB_GEMM_DGRAD: return p0.T >= 32 && (p0.ldb % 4) == 0 && (p0.ldx % 4) == 0;
    case DIB_GEMM_WGRAD: return (p0.lda % 32) == 0 && (p0.ldb % 32) == 0 && (p0.ldc % 4) == 0;
  }
  return false;
}

namespace {

// one launch over problems hp[0 .. L.nprob) (L.probs: their device copies); the TMA maps start at hp[0]
cudaError_t launch_group(int mode, const DibGemmLaunch& L, const DibGemmProblem* hp, cudaStream_t st) {
  const DibGemmProblem& p0 = hp[0];
  const int nf = L.nprob;
  const long long sa = nf > 1 ? hp[1].a_off - hp[0].a_off : 0, sb = nf > 1 ? hp[1].b_off - hp[0].b_off : 0;
  const int BN = (p0.C % 128 == 0) ? 128 : 64;
  CUtensorMap mapA, mapB;
  bool ok = true;
  const float* A = L.baseA + p0.a_off;
  const float* B = L.baseB + p0.b_off;
  switch (mode) {      // TMA maps of the K-major operands (MN-major ones are loaded by the producer warpgroup)
    case DIB_GEMM_FWD:    // A: h [M x lda] K-major; B: W [T x C] MN-major
      ok = make_map_kmajor(&mapA, A, p0.lda, L.M, p0.lda, sa, nf, kBM);
      mapB = mapA;
      break;
    case DIB_GEMM_DGRAD:  // A: dz [M x lda] K-major; B: W [C rows x T] K-major
      ok = make_map_kmajor(&mapA, A, p0.lda, L.M, p0.lda, sa, nf, kBM) &&
           make_map_kmajor(&mapB, B, p0.ldb, p0.C, p0.ldb, sb, nf, BN);
      break;
    default:              // A: h [m x lda] MN-major; B: dz [m x ldb] MN-major
      memset(&mapA, 0, sizeof(mapA));
      mapB = mapA;
      break;
  }
  if (!ok) return cudaErrorInvalidValue;
#define DIB_TC_CASE(MODE)                                                           \
  case MODE:                                                                        \
    return BN == 128 ? launch_tc<MODE, 128>(L, mapA, mapB, st) : launch_tc<MODE, 64>(L, mapA, mapB, st);
  switch (mode) {
    DIB_TC_CASE(DIB_GEMM_FWD)
    DIB_TC_CASE(DIB_GEMM_DGRAD)
    DIB_TC_CASE(DIB_GEMM_WGRAD)
  }
#undef DIB_TC_CASE
  return cudaErrorInvalidValue;
}

}  // namespace

cudaError_t dib_launch_gemm_tc(int mode, const DibGemmLaunch& L, const DibGemmProblem* hp, cudaStream_t st) {
  // gridDim.z holds (problem, split): a group with more than 65 535 of them runs as consecutive launches over its problems,
  // each with TMA maps built from its own first descriptor (the kernel's problem index is relative to the launch)
  const int chunk = dib_gemm_chunk_problems(L.nprob, mode == DIB_GEMM_WGRAD ? L.nsplit : 1);
  if (L.nprob > 0 && chunk < 1) return cudaErrorInvalidConfiguration;
  for (int first = 0; first < L.nprob; first += chunk) {
    DibGemmLaunch part = L;
    part.probs = L.probs + first;
    part.nprob = L.nprob - first < chunk ? L.nprob - first : chunk;
    const cudaError_t e = launch_group(mode, part, hp + first, st);
    if (e != cudaSuccess) return e;
  }
  return cudaSuccess;
}
