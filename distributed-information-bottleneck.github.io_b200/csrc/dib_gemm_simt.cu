// dib_gemm_simt.cu -- grouped FP32 (CUDA-core FMA) GEMMs with fused epilogues: the exact-fp32 parity path
// for every dense contraction of the Distributed-IB step, batched over the F independent feature encoders
// (the reference unrolls them into F separate sub-graphs, models.py:105-106).
//
// Canonical form  Out[R x C] = sum_t Aop[R x T] * Bop[T x C]  with three modes:
//   FWD   h_k  = act(h_{k-1} W_k + b_k)            R = batch rows, T = fan-in,  C = fan-out   (models.py:76-77)
//   DGRAD dz_{k-1} = (dz_k W_k^T) * act'(h_{k-1})  R = batch rows, T = fan-out, C = fan-in    (GradientTape)
//   WGRAD dW_k = h_{k-1}^T dz_k, db_k = colsum dz_k over one batch slice -> deterministic split partials
// Invariants kept by dib_api.cu: every activation/gradient buffer has a leading dimension that is a multiple
// of 4 floats, is 16-byte aligned, and its pad columns are written as zeros by the producing kernel.
#include "dib_common.cuh"
#include "dib_kernels.h"

namespace {

template <int W>
__device__ __forceinline__ void ld_frag(const float* p, float* out) {
  if constexpr (W == 4) {
    const float4 v = *reinterpret_cast<const float4*>(p);
    out[0] = v.x; out[1] = v.y; out[2] = v.z; out[3] = v.w;
  } else if constexpr (W == 2) {
    const float2 v = *reinterpret_cast<const float2*>(p);
    out[0] = v.x; out[1] = v.y;
  } else {
    out[0] = p[0];
  }
}

template <int MODE, int BR, int BC, int BT, int TM, int TN>
__global__ void __launch_bounds__((BR / TM) * (BC / TN))
dib_gemm_simt_kernel(const DibGemmProblem* __restrict__ probs, const float* __restrict__ baseA,
                     const float* __restrict__ baseB, float* __restrict__ baseC, float* baseX,
                     int M, int nsplit, int rows_per_split, long long split_stride, float alpha, int round_out) {
  constexpr int TX = BC / TN, TY = BR / TM, NT = TX * TY;
  constexpr int CM = TM >= 4 ? 4 : TM, NCM = TM / CM;   // row chunks of the per-thread micro tile
  constexpr int CN = TN >= 4 ? 4 : TN, NCN = TN / CN;   // column chunks
  constexpr int LDA_S = BR + 4, LDB_S = BC + 4;
  constexpr int A_VEC = BT * BR / 4, A_PER = (A_VEC + NT - 1) / NT;
  constexpr int B_VEC = BT * BC / 4, B_PER = (B_VEC + NT - 1) / NT;
  static_assert(BT % 4 == 0 && BR % 4 == 0 && BC % 4 == 0, "tile dims");

  __shared__ __align__(16) float As[2][BT][LDA_S];
  __shared__ __align__(16) float Bs[2][BT][LDB_S];

  const int tid = threadIdx.x, tx = tid % TX, ty = tid / TX;
  int prob, split = 0, r0, c0;
  if constexpr (MODE == DIB_GEMM_WGRAD) {
    prob = blockIdx.z / nsplit; split = blockIdx.z % nsplit;
    c0 = blockIdx.x * BC; r0 = blockIdx.y * BR;
  } else {
    prob = blockIdx.z; r0 = blockIdx.x * BR; c0 = blockIdx.y * BC;
  }
  const DibGemmProblem p = probs[prob];
  const int R = (MODE == DIB_GEMM_WGRAD) ? p.R : M;
  const int C = p.C;
  int t_begin = 0, t_end = p.T;
  if constexpr (MODE == DIB_GEMM_WGRAD) {
    t_begin = split * rows_per_split;
    t_end = min(M, t_begin + rows_per_split);
  }
  if (r0 >= R || c0 >= C) return;   // uniform per block
  const float* __restrict__ A = baseA + p.a_off;
  const float* __restrict__ B = baseB + p.b_off;
  const int lda = p.lda, ldb = p.ldb;
  const bool vecB = ((ldb & 3) == 0) && ((reinterpret_cast<uintptr_t>(B) & 15) == 0);

  float4 ra[A_PER], rb[B_PER];

  auto load_tiles = [&](int t0) {   // t0 is absolute
#pragma unroll
    for (int i = 0; i < A_PER; ++i) {
      const int v = tid + i * NT;
      float4 val = make_float4(0.f, 0.f, 0.f, 0.f);
      if (A_VEC % NT == 0 || v < A_VEC) {
        if constexpr (MODE == DIB_GEMM_WGRAD) {      // Aop[r][t] = A[t*lda + r]   (r contiguous)
          const int t = v / (BR / 4), r4 = (v % (BR / 4)) * 4;
          if (t0 + t < t_end && r0 + r4 < lda)
            val = *reinterpret_cast<const float4*>(A + (long long)(t0 + t) * lda + r0 + r4);
        } else {                                      // Aop[r][t] = A[r*lda + t]   (t contiguous)
          const int r = v / (BT / 4), t4 = (v % (BT / 4)) * 4;
          if (r0 + r < R && t0 + t4 < t_end && t0 + t4 < lda)
            val = *reinterpret_cast<const float4*>(A + (long long)(r0 + r) * lda + t0 + t4);
        }
      }
      ra[i] = val;
    }
#pragma unroll
    for (int i = 0; i < B_PER; ++i) {
      const int v = tid + i * NT;
      float4 val = make_float4(0.f, 0.f, 0.f, 0.f);
      if (B_VEC % NT == 0 || v < B_VEC) {
        if constexpr (MODE == DIB_GEMM_DGRAD) {       // Bop[t][c] = W[c*ldb + t]   (t contiguous)
          const int c = v / (BT / 4), t4 = (v % (BT / 4)) * 4;
          if (c0 + c < C) {
            const float* src = B + (long long)(c0 + c) * ldb + t0 + t4;
            if (vecB) {
              if (t0 + t4 < t_end) val = *reinterpret_cast<const float4*>(src);
            } else {
              if (t0 + t4 + 0 < t_end) val.x = src[0];
              if (t0 + t4 + 1 < t_end) val.y = src[1];
              if (t0 + t4 + 2 < t_end) val.z = src[2];
              if (t0 + t4 + 3 < t_end) val.w = src[3];
            }
          }
        } else {                                      // Bop[t][c] = B[t*ldb + c]   (c contiguous)
          const int t = v / (BC / 4), c4 = (v % (BC / 4)) * 4;
          if (t0 + t < t_end) {
            const float* src = B + (long long)(t0 + t) * ldb + c0 + c4;
            if (vecB) {
              if (c0 + c4 < ldb) val = *reinterpret_cast<const float4*>(src);
            } else {
              if (c0 + c4 + 0 < C) val.x = src[0];
              if (c0 + c4 + 1 < C) val.y = src[1];
              if (c0 + c4 + 2 < C) val.z = src[2];
              if (c0 + c4 + 3 < C) val.w = src[3];
            }
          }
        }
      }
      rb[i] = val;
    }
  };

  auto store_tiles = [&](int buf) {
#pragma unroll
    for (int i = 0; i < A_PER; ++i) {
      const int v = tid + i * NT;
      if (A_VEC % NT == 0 || v < A_VEC) {
        if constexpr (MODE == DIB_GEMM_WGRAD) {
          const int t = v / (BR / 4), r4 = (v % (BR / 4)) * 4;
          *reinterpret_cast<float4*>(&As[buf][t][r4]) = ra[i];
        } else {
          const int r = v / (BT / 4), t4 = (v % (BT / 4)) * 4;
          As[buf][t4 + 0][r] = ra[i].x; As[buf][t4 + 1][r] = ra[i].y;
          As[buf][t4 + 2][r] = ra[i].z; As[buf][t4 + 3][r] = ra[i].w;
        }
      }
    }
#pragma unroll
    for (int i = 0; i < B_PER; ++i) {
      const int v = tid + i * NT;
      if (B_VEC % NT == 0 || v < B_VEC) {
        if constexpr (MODE == DIB_GEMM_DGRAD) {
          const int c = v / (BT / 4), t4 = (v % (BT / 4)) * 4;
          Bs[buf][t4 + 0][c] = rb[i].x; Bs[buf][t4 + 1][c] = rb[i].y;
          Bs[buf][t4 + 2][c] = rb[i].z; Bs[buf][t4 + 3][c] = rb[i].w;
        } else {
          const int t = v / (BC / 4), c4 = (v % (BC / 4)) * 4;
          *reinterpret_cast<float4*>(&Bs[buf][t][c4]) = rb[i];
        }
      }
    }
  };

  float acc[TM][TN];
#pragma unroll
  for (int i = 0; i < TM; ++i)
#pragma unroll
    for (int j = 0; j < TN; ++j) acc[i][j] = 0.f;
  float bsum[TN];
#pragma unroll
  for (int j = 0; j < TN; ++j) bsum[j] = 0.f;
  const bool do_bsum = (MODE == DIB_GEMM_WGRAD) && (blockIdx.y == 0) && (ty == 0);

  const int ntiles = DIB_CEIL_DIV(t_end - t_begin, BT);
  if (ntiles > 0) {
    load_tiles(t_begin);
    store_tiles(0);
  }
  __syncthreads();
  for (int it = 0; it < ntiles; ++it) {
    const int buf = it & 1;
    if (it + 1 < ntiles) load_tiles(t_begin + (it + 1) * BT);
#pragma unroll
    for (int kk = 0; kk < BT; ++kk) {
      float a[TM], b[TN];
#pragma unroll
      for (int ch = 0; ch < NCM; ++ch) ld_frag<CM>(&As[buf][kk][ch * (BR / NCM) + ty * CM], &a[ch * CM]);
#pragma unroll
      for (int ch = 0; ch < NCN; ++ch) ld_frag<CN>(&Bs[buf][kk][ch * (BC / NCN) + tx * CN], &b[ch * CN]);
#pragma unroll
      for (int i = 0; i < TM; ++i)
#pragma unroll
        for (int j = 0; j < TN; ++j) acc[i][j] = fmaf(a[i], b[j], acc[i][j]);
      if constexpr (MODE == DIB_GEMM_WGRAD) {
        if (do_bsum) {
#pragma unroll
          for (int j = 0; j < TN; ++j) bsum[j] += b[j];
        }
      }
    }
    if (it + 1 < ntiles) store_tiles(buf ^ 1);
    __syncthreads();
  }

  // ------------------------------------------------------------------ epilogue
  float* __restrict__ Out = baseC + p.c_off + (MODE == DIB_GEMM_WGRAD ? (long long)split * split_stride : 0ll);
  const int ldc = p.ldc;
  const bool vecC = ((ldc & 3) == 0) && ((reinterpret_cast<uintptr_t>(Out) & 15) == 0);
#pragma unroll
  for (int i = 0; i < TM; ++i) {
    const int r = r0 + (i / CM) * (BR / NCM) + ty * CM + (i % CM);
    if (r >= R) continue;
#pragma unroll
    for (int ch = 0; ch < NCN; ++ch) {
      const int c = c0 + ch * (BC / NCN) + tx * CN;
      float vals[CN];
#pragma unroll
      for (int j = 0; j < CN; ++j) {
        float v = acc[i][ch * CN + j];
        const int cc = c + j;
        if constexpr (MODE == DIB_GEMM_FWD) {
          if (cc < C) v = dib_act(p.act, v + (baseB + p.x_off)[cc], alpha);
        } else if constexpr (MODE == DIB_GEMM_DGRAD) {
          if (cc < C && p.act != DIB_ACT_LINEAR) v *= dib_act_grad(p.act, (baseX + p.x_off)[(long long)r * p.ldx + cc], alpha);
        }
        if constexpr (MODE != DIB_GEMM_WGRAD) v = dib_maybe_round(v, round_out);
        vals[j] = cc < C ? v : 0.f;
      }
      float* dst = Out + (long long)r * ldc + c;
      if (CN == 4 && vecC && c + 4 <= ldc) {
        *reinterpret_cast<float4*>(dst) = make_float4(vals[0], vals[1], vals[2], vals[3]);
      } else {
#pragma unroll
        for (int j = 0; j < CN; ++j)
          if (c + j < ldc) dst[j] = vals[j];
      }
    }
  }
  if constexpr (MODE == DIB_GEMM_WGRAD) {
    if (do_bsum && p.x_off >= 0) {
      float* db = baseX + p.x_off + (long long)split * split_stride;
#pragma unroll
      for (int ch = 0; ch < NCN; ++ch)
#pragma unroll
        for (int j = 0; j < CN; ++j) {
          const int cc = c0 + ch * (BC / NCN) + tx * CN + j;
          if (cc < C) db[cc] = bsum[ch * CN + j];
        }
    }
  }
}

template <int MODE, int BR, int BC, int BT, int TM, int TN>
cudaError_t launch_cfg(const DibGemmLaunch& L, cudaStream_t st) {
  constexpr int NT = (BR / TM) * (BC / TN);
  // gridDim.z holds (problem, split): a group with more than 65 535 of them runs as consecutive launches over its problems
  const int zper = MODE == DIB_GEMM_WGRAD ? L.nsplit : 1;
  const int chunk = dib_gemm_chunk_problems(L.nprob, zper);
  if (L.nprob > 0 && chunk < 1) return cudaErrorInvalidConfiguration;
  for (int first = 0; first < L.nprob; first += chunk) {
    const int np = L.nprob - first < chunk ? L.nprob - first : chunk;
    dim3 grid;
    if (MODE == DIB_GEMM_WGRAD)
      grid = dim3(DIB_CEIL_DIV(L.maxC, BC), DIB_CEIL_DIV(L.maxR, BR), np * L.nsplit);
    else
      grid = dim3(DIB_CEIL_DIV(L.M, BR), DIB_CEIL_DIV(L.maxC, BC), np);
    if (grid.x == 0 || grid.y == 0 || grid.z == 0) return cudaSuccess;
    dib_gemm_simt_kernel<MODE, BR, BC, BT, TM, TN><<<grid, NT, 0, st>>>(
        L.probs + first, L.baseA, L.baseB, L.baseC, L.baseX, L.M, L.nsplit, L.rows_per_split, L.split_stride, L.alpha,
        L.round_out);
    dib_note_launch();
    const cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) return e;
  }
  return cudaSuccess;
}

template <int MODE>
cudaError_t launch_mode(const DibGemmLaunch& L, cudaStream_t st) {
  if (MODE == DIB_GEMM_WGRAD && L.maxR <= 32) {
    if (L.maxC > 64) return launch_cfg<MODE, 16, 128, 32, 2, 4>(L, st);
    return launch_cfg<MODE, 16, 64, 32, 1, 4>(L, st);
  }
  if (L.maxC > 64) return launch_cfg<MODE, 128, 128, 8, 8, 8>(L, st);
  if (L.maxC > 16) return launch_cfg<MODE, 128, 64, 8, 8, 4>(L, st);
  return launch_cfg<MODE, 128, 16, 16, 4, 2>(L, st);
}

}  // namespace

cudaError_t dib_launch_gemm_simt(int mode, const DibGemmLaunch& L, cudaStream_t st) {
  switch (mode) {
    case DIB_GEMM_FWD: return launch_mode<DIB_GEMM_FWD>(L, st);
    case DIB_GEMM_DGRAD: return launch_mode<DIB_GEMM_DGRAD>(L, st);
    case DIB_GEMM_WGRAD: return launch_mode<DIB_GEMM_WGRAD>(L, st);
  }
  return cudaErrorInvalidValue;
}
