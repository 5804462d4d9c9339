// dib_test_hooks.cu -- the unit-test hooks declared in include/dib_b200_test_hooks.h: each launches one kernel family
// through the launcher the library's own steps use, after checking every argument on the host, and synchronises the stream.
#include <algorithm>
#include <cmath>
#include <cstddef>
#include <vector>

#include "dib_common.cuh"
#include "dib_kernels.h"
#include "../../include/dib_b200_test_hooks.h"

namespace {
// the memory contracts of the 16-bit kernels: TMA descriptors need 16-byte bases and row pitches, and the epilogues store and
// load whole column pairs (4 bytes) or 8-column vectors (16 bytes)
std::string int16_base_error(const char* name, const void* p) {
  return p && reinterpret_cast<uintptr_t>(p) % 16 ? std::string(name) + " must be 16-byte aligned" : std::string();
}
std::string int16_ld_error(const char* name, int64_t ld, int64_t width) {
  if (ld % 8 || ld < width)
    return std::string(name) + " must be a multiple of 8 and >= " + std::to_string(width) + " (" + name + " = " +
           std::to_string(ld) + ")";
  return std::string();
}
std::string int16_bias_error(const char* name, const float* p) {
  return p && reinterpret_cast<uintptr_t>(p) % 8 ? std::string(name) + " must be 8-byte aligned" : std::string();
}
bool known_act(int32_t act) { return act >= DIB_ACT_LINEAR && act <= DIB_ACT_ELU; }
int sync_result(const std::string& fn, cudaError_t e, cudaStream_t st) {
  const cudaError_t es = cudaStreamSynchronize(st);
  if (e != cudaSuccess) return fail(fn + "launch: " + cudaGetErrorString(e));
  if (es != cudaSuccess) return fail(fn + "sync: " + cudaGetErrorString(es));
  return 0;
}
}  // namespace

// returns fail(fn + the message) unless the check's message is empty
#define DIB_HOOK_CHECK(msg)                          \
  do {                                               \
    const std::string _m = (msg);                    \
    if (!_m.empty()) return fail(fn + _m);           \
  } while (0)

extern "C" {

// the header's C mirror of the kernels' problem descriptor: the test hook hands its array to the kernels as it is
static_assert(sizeof(dib_gemm_problem) == sizeof(DibGemmProblem), "dib_gemm_problem size");
static_assert(offsetof(dib_gemm_problem, a_off) == offsetof(DibGemmProblem, a_off) &&
              offsetof(dib_gemm_problem, x_off) == offsetof(DibGemmProblem, x_off) &&
              offsetof(dib_gemm_problem, lda) == offsetof(DibGemmProblem, lda) &&
              offsetof(dib_gemm_problem, ldx) == offsetof(DibGemmProblem, ldx) &&
              offsetof(dib_gemm_problem, T) == offsetof(DibGemmProblem, T) &&
              offsetof(dib_gemm_problem, C) == offsetof(DibGemmProblem, C) &&
              offsetof(dib_gemm_problem, R) == offsetof(DibGemmProblem, R) &&
              offsetof(dib_gemm_problem, act) == offsetof(DibGemmProblem, act), "dib_gemm_problem layout");

// one grouped GEMM launch of the simt or tc kernel, set up as gemm() sets up its launches (unit tests)
int dib_debug_gemm(int32_t kernel, int32_t mode, const dib_gemm_problem* problems, int32_t nprob, const float* A,
                   const float* B, float* C, float* X, const float* bias, int32_t M, int32_t maxC, int32_t maxR, int32_t nsplit,
                   int32_t rows_per_split, int64_t split_stride, float alpha, int32_t round_out, void* stream) {
  const std::string fn = "dib_debug_gemm: ";
  if (kernel != DIB_GEMM_KERNEL_SIMT && kernel != DIB_GEMM_KERNEL_TC) return fail(fn + "unknown kernel");
  if (mode < DIB_GEMM_FWD || mode > DIB_GEMM_WGRAD) return fail(fn + "unknown mode");
  if (!problems || nprob < 1 || M < 0 || nsplit < 1) return fail(fn + "needs nprob >= 1, M >= 0 and nsplit >= 1");
  if (kernel == DIB_GEMM_KERNEL_SIMT && mode == DIB_GEMM_FWD && bias && bias != B)
    return fail(fn + "the simt kernel reads FWD biases from B's base (bias must be B or null)");
  const DibGemmProblem* hp = reinterpret_cast<const DibGemmProblem*>(problems);
  const cudaStream_t st = static_cast<cudaStream_t>(stream);
  if (kernel == DIB_GEMM_KERNEL_TC && !dib_gemm_tc_eligible(mode, hp, nprob, nullptr))
    return fail(fn + "the tensor-core kernel cannot run this group");
  DibGemmProblem* dp = nullptr;
  DIB_CUDA_OK(cudaMalloc(&dp, (size_t)nprob * sizeof(DibGemmProblem)));
  cudaError_t e = cudaMemcpy(dp, hp, (size_t)nprob * sizeof(DibGemmProblem), cudaMemcpyHostToDevice);
  DibGemmLaunch L;
  L.probs = dp; L.nprob = nprob; L.baseA = A; L.baseB = B; L.baseC = C; L.baseX = X; L.M = M;
  L.maxC = maxC; L.maxR = maxR; L.nsplit = nsplit; L.rows_per_split = rows_per_split;
  L.split_stride = split_stride; L.alpha = alpha; L.round_out = round_out ? 1 : 0;
  if (mode == DIB_GEMM_FWD) L.baseBias = bias;
  if (e == cudaSuccess)
    e = kernel == DIB_GEMM_KERNEL_TC ? dib_launch_gemm_tc(mode, L, hp, st) : dib_launch_gemm_simt(mode, L, st);
  const int r = sync_result(fn, e, st);
  cudaFree(dp);
  return r;
}

// the streaming InfoNCE sweeps with the arguments infonce_args fills, through the launchers the steps use (unit tests)
int dib_debug_infonce_stream(int32_t kind, float temperature, const float* e1, int32_t ld1, const float* e2, int32_t ld2,
                             int64_t n, int32_t d, int64_t row0, int64_t rows, float* lse_r, float* lse_c, int32_t lse_stride,
                             float* diag, float* loss_sum, float* d_e1, int32_t ld_d1, float* d_e2, int32_t ld_d2,
                             int32_t round_out, int32_t phases, void* stream) {
  const char* fn = "dib_debug_infonce_stream: ";
  if (kind < 0 || kind > 4) return fail(std::string(fn) + "unknown similarity kind " + std::to_string(kind));
  if (!(temperature > 0.f) || !std::isfinite(temperature)) return fail(std::string(fn) + "needs 0 < temperature < inf");
  if (d < 1 || d > 512) return fail(std::string(fn) + "needs 1 <= d <= 512 (d = " + std::to_string(d) + ")");
  if (ld1 < d || ld2 < d) return fail(std::string(fn) + "needs ld1, ld2 >= d");
  if (n < 1 || n > 0x7fffffffll) return fail(std::string(fn) + "needs 1 <= n < 2^31 (n = " + std::to_string(n) + ")");
  if (row0 < 0 || rows < 1 || row0 + rows > n)
    return fail(std::string(fn) + "the own rows [row0, row0 + rows) must be a nonempty range inside [0, n) (row0 = " +
                std::to_string(row0) + ", rows = " + std::to_string(rows) + ", n = " + std::to_string(n) + ")");
  if (lse_stride < 1) return fail(std::string(fn) + "needs lse_stride >= 1");
  if (phases < 1 || phases > 3) return fail(std::string(fn) + "phases is a mask of 1 (loss sweeps) and 2 (gradient sweeps)");
  if (!e1 || !e2 || !lse_r || !lse_c) return fail(std::string(fn) + "e1, e2, lse_r and lse_c must not be null");
  if ((phases & 1) && (!diag || !loss_sum)) return fail(std::string(fn) + "the loss sweeps need diag and loss_sum");
  if ((phases & 2) && ((d_e1 && ld_d1 < d) || (d_e2 && ld_d2 < d))) return fail(std::string(fn) + "needs ld_d1, ld_d2 >= d");
  DibInfonceStream a;
  a.kind = kind; a.temperature = temperature;
  a.e1 = e1; a.ld1 = ld1;
  a.e2 = e2; a.ld2 = ld2;
  a.n = n; a.d = d;
  a.row0 = row0; a.rows = rows;
  a.lse_r = lse_r; a.lse_c = lse_c; a.lse_stride = lse_stride;
  a.diag = diag; a.loss_sum = loss_sum; a.acc_zero = nullptr;
  a.d_e1 = d_e1; a.ld_d1 = ld_d1;
  a.d_e2 = d_e2; a.ld_d2 = ld_d2;
  a.round_out = round_out ? 1 : 0;
  const cudaStream_t st = static_cast<cudaStream_t>(stream);
  cudaError_t e = cudaSuccess;
  if (phases & 1) e = dib_launch_infonce_stream_loss(a, st);
  if (e == cudaSuccess && (phases & 2)) e = dib_launch_infonce_stream_grads(a, st);
  return sync_result(fn, e, st);
}

// the attention core of a set-transformer block, fixed-size or key-tiled, through the launchers the steps use (unit tests)
int dib_debug_set_attention(int32_t variable_sizes, int32_t phases, const float* q, const float* k, const float* v,
                            const float* dout, int32_t ld, int64_t sets, int32_t heads, int32_t L, int32_t dk,
                            const int32_t* set_sizes, float* o, float* lse, float* dq, float* dk_, float* dv, float* dsum,
                            int32_t round_out, void* stream) {
  const std::string fn = "dib_debug_set_attention: ";
  if (variable_sizes != 0 && variable_sizes != 1) return fail(fn + "variable_sizes is 0 (fixed-size kernels) or 1 (key-tiled)");
  if (phases < 1 || phases > 3) return fail(fn + "phases is a mask of 1 (forward) and 2 (backward)");
  const int maxL = dib_attn_max_set_size(variable_sizes);
  if (L < 1 || L > maxL) return fail(fn + "needs 1 <= L <= " + std::to_string(maxL) + " (L = " + std::to_string(L) + ")");
  if (!dib_attn_heads_ok(heads, dk))
    return fail(fn + "needs heads >= 1, 1 <= dk <= 128 and heads * dk a multiple of 4 (heads = " + std::to_string(heads) +
                ", dk = " + std::to_string(dk) + ")");
  if ((int64_t)ld < (int64_t)heads * dk) return fail(fn + "needs ld >= heads * dk (ld = " + std::to_string(ld) + ")");
  if (sets < 0 || sets > 65535) return fail(fn + "needs 0 <= sets <= 65535 (sets = " + std::to_string(sets) + ")");
  if (!q || !k || !v || !o || !lse) return fail(fn + "q, k, v, o and lse must not be null");
  if ((phases & 2) && (!dout || !dq || !dk_ || !dv)) return fail(fn + "the backward needs dout, dq, dk and dv");
  if (variable_sizes && !set_sizes) return fail(fn + "the key-tiled kernels need set_sizes");
  if (variable_sizes && (phases & 2) && !dsum) return fail(fn + "the key-tiled backward needs dsum");
  DibAttnArgs a;
  a.q = q; a.k = k; a.v = v; a.ld = ld;
  a.o = o; a.lse = lse;
  a.sets = sets; a.heads = heads; a.L = L; a.dk = dk;
  a.round_out = round_out ? 1 : 0;
  a.dout = dout; a.dq = dq; a.dk_ = dk_; a.dv = dv;
  a.set_sizes = variable_sizes ? set_sizes : nullptr; a.dsum = variable_sizes ? dsum : nullptr;
  DIB_CUDA_OK(variable_sizes ? dib_attn_varlen_prepare() : dib_attn_prepare());
  const cudaStream_t st = static_cast<cudaStream_t>(stream);
  cudaError_t e = cudaSuccess;
  if (phases & 1) e = variable_sizes ? dib_launch_attn_varlen_fwd(a, st) : dib_launch_attn_fwd(a, st);
  if (e == cudaSuccess && (phases & 2)) e = variable_sizes ? dib_launch_attn_varlen_bwd(a, st) : dib_launch_attn_bwd(a, st);
  return sync_result(fn, e, st);
}

// LayerNorm(a + b) forward and / or backward of a set-transformer block, set up as forward_set_blocks / backward_set_blocks
// set them up (unit tests)
int dib_debug_layer_norm(int32_t phases, const float* a, const float* b, int32_t ld, int64_t rows, int32_t E, const float* gamma,
                         const float* beta, float epsilon, float* y, float* mean, float* rstd, const float* dy0,
                         const float* dy1, const float* dy2, const float* dy3, const float* dy_pool, int32_t pool_rows,
                         const int32_t* set_sizes, float* d_res, float* d_branch, int32_t branch_act, float alpha, float* part,
                         int64_t split_stride, int64_t gamma_off, int64_t beta_off, int32_t nsplit, int64_t rows_per_split,
                         int32_t round_out, void* stream) {
  const std::string fn = "dib_debug_layer_norm: ";
  if (phases < 1 || phases > 3) return fail(fn + "phases is a mask of 1 (forward) and 2 (backward)");
  if (!dib_set_width_ok(E)) return fail(fn + "needs 1 <= E <= 128, a multiple of 4 (E = " + std::to_string(E) + ")");
  if (ld < E) return fail(fn + "needs ld >= E (ld = " + std::to_string(ld) + ")");
  if (rows < 0) return fail(fn + "needs rows >= 0");
  if (!(epsilon >= 0.f) || !std::isfinite(epsilon)) return fail(fn + "needs 0 <= epsilon < inf");
  if (!a || !b || !gamma || !mean || !rstd) return fail(fn + "a, b, gamma, mean and rstd must not be null");
  if ((phases & 1) && (!beta || !y)) return fail(fn + "the forward needs beta and y");
  DibLayerNorm l;
  l.a = a; l.b = b; l.ld = ld; l.rows = rows; l.E = E;
  l.gamma = gamma; l.beta = beta; l.epsilon = epsilon;
  l.y = y; l.mean = mean; l.rstd = rstd;
  l.round_out = round_out ? 1 : 0;
  DibLayerNormBwd g;
  if (phases & 2) {
    if (!d_res || !part) return fail(fn + "the backward needs d_res and part");
    if (nsplit < 1 || rows_per_split < 1 || (int64_t)nsplit * rows_per_split < rows)
      return fail(fn + "needs nsplit >= 1, rows_per_split >= 1 and nsplit * rows_per_split >= rows");
    if (gamma_off < 0 || beta_off < 0 || gamma_off + E > split_stride || beta_off + E > split_stride)
      return fail(fn + "the d gamma / d beta partial ranges [gamma_off, gamma_off + E), [beta_off, beta_off + E) must lie "
                       "inside [0, split_stride)");
    if (dy_pool && pool_rows < 1) return fail(fn + "dy_pool needs pool_rows >= 1");
    if (set_sizes && !dy_pool) return fail(fn + "set_sizes needs dy_pool");
    if (d_branch && (branch_act < DIB_ACT_LINEAR || branch_act > DIB_ACT_ELU)) return fail(fn + "unknown branch_act");
    g.dy[0] = dy0; g.dy[1] = dy1; g.dy[2] = dy2; g.dy[3] = dy3;
    g.dy_pool = dy_pool; g.pool_rows = pool_rows; g.pool_scale = dy_pool ? 1.f / (float)pool_rows : 0.f; g.set_sizes = set_sizes;
    g.d_res = d_res; g.d_branch = d_branch; g.branch_act = branch_act; g.alpha = alpha;
    g.part = part; g.split_stride = split_stride; g.gamma_off = gamma_off; g.beta_off = beta_off;
    g.nsplit = nsplit; g.rows_per_split = rows_per_split;
  }
  const cudaStream_t st = static_cast<cudaStream_t>(stream);
  cudaError_t e = cudaSuccess;
  if (phases & 1) e = dib_launch_ln_fwd(l, st);
  if (e == cudaSuccess && (phases & 2)) e = dib_launch_ln_bwd(l, g, st);
  return sync_result(fn, e, st);
}

// the mean over each set's rows (fixed or variable sizes) or zero_pad_rows, through the launchers the steps use (unit tests)
int dib_debug_set_pool(int32_t zero_pad, float* x, int32_t ld, int32_t E, int32_t L, int64_t sets, const int32_t* set_sizes,
                       float* out, int32_t ldo, int32_t round_out, void* stream) {
  const std::string fn = "dib_debug_set_pool: ";
  const int maxL = dib_attn_max_set_size(set_sizes != nullptr);
  if (zero_pad != 0 && zero_pad != 1) return fail(fn + "zero_pad is 0 (mean pooling) or 1 (zero_pad_rows)");
  if (zero_pad && !set_sizes) return fail(fn + "zero_pad_rows needs set_sizes");
  if (L < 1 || L > maxL) return fail(fn + "needs 1 <= L <= " + std::to_string(maxL) + " (L = " + std::to_string(L) + ")");
  if (sets < 0 || sets > 65535) return fail(fn + "needs 0 <= sets <= 65535 (sets = " + std::to_string(sets) + ")");
  if (!x) return fail(fn + "x must not be null");
  if (!zero_pad && (!dib_set_width_ok(E) || ld < E || ldo < E || !out))
    return fail(fn + "mean pooling needs 1 <= E <= 128 a multiple of 4, ld >= E, ldo >= E and out");
  if (zero_pad && ld < 1) return fail(fn + "needs ld >= 1");
  const cudaStream_t st = static_cast<cudaStream_t>(stream);
  cudaError_t e;
  if (zero_pad) e = dib_launch_zero_pad_rows(x, ld, sets * L, L, set_sizes, st);
  else if (set_sizes) e = dib_launch_pool_varlen_fwd(x, ld, E, L, sets, set_sizes, out, ldo, round_out ? 1 : 0, st);
  else e = dib_launch_pool_fwd(x, ld, E, L, sets, out, ldo, round_out ? 1 : 0, st);
  return sync_result(fn, e, st);
}

// the reparameterisation forward and / or backward, set up as reparam_args sets them up (unit tests)
int dib_debug_reparam(int32_t phases, const float* enc_out, int64_t feat_stride, int32_t ldo, int32_t F, int32_t E, int64_t n,
                      const float* eps, uint64_t seed, uint32_t step, const uint32_t* step_dev, uint64_t sample_offset,
                      const int32_t* set_sizes, int32_t set_len, float* emb, int32_t ldemb, float* user_emb, float* kl_part,
                      int32_t nblk_stride, const float* d_emb, const float* beta_dev, float inv_batch, float* d_out,
                      int32_t round_out, void* stream) {
  const std::string fn = "dib_debug_reparam: ";
  if (phases < 1 || phases > 3) return fail(fn + "phases is a mask of 1 (forward) and 2 (backward)");
  if (F < 1 || F > 65535) return fail(fn + "needs 1 <= F <= 65535 (F = " + std::to_string(F) + ")");
  if (E < 1) return fail(fn + "needs E >= 1");
  if ((int64_t)ldo < 2 * (int64_t)E) return fail(fn + "needs ldo >= 2E (ldo = " + std::to_string(ldo) + ")");
  if (n < 0 || n > 0x7fffffffll) return fail(fn + "needs 0 <= n < 2^31 (n = " + std::to_string(n) + ")");
  if (feat_stride < n * ldo) return fail(fn + "needs feat_stride >= n * ldo");
  if (!enc_out) return fail(fn + "enc_out must not be null");
  if (set_sizes && (set_len < 1 || set_len > DIB_MAX_VARIABLE_SET_SIZE || n % set_len))
    return fail(fn + "set_sizes needs 1 <= set_len <= " + std::to_string(DIB_MAX_VARIABLE_SET_SIZE) + " dividing n (set_len = " +
                std::to_string(set_len) + ")");
  if ((int64_t)ldemb < (int64_t)F * E) return fail(fn + "needs ldemb >= F * E (ldemb = " + std::to_string(ldemb) + ")");
  if ((phases & 1) && (!emb || !kl_part)) return fail(fn + "the forward needs emb and kl_part");
  if ((phases & 1) && (int64_t)nblk_stride < (n + 255) / 256) return fail(fn + "needs nblk_stride >= ceil(n / 256)");
  if ((phases & 2) && (!d_emb || !beta_dev || !d_out)) return fail(fn + "the backward needs d_emb, beta_dev and d_out");
  DibReparamArgs a;
  a.enc_out = enc_out; a.feat_stride = feat_stride; a.ldo = ldo;
  a.eps = eps; a.seed = seed; a.step = step; a.step_dev = step_dev; a.sample_offset = sample_offset;
  a.F = F; a.E = E; a.n = n; a.round_out = round_out ? 1 : 0;
  a.set_sizes = set_sizes; a.set_len = set_sizes ? set_len : 1;
  const cudaStream_t st = static_cast<cudaStream_t>(stream);
  cudaError_t e = cudaSuccess;
  if (phases & 1) e = dib_launch_reparam_fwd(a, emb, ldemb, user_emb, kl_part, nblk_stride, st);
  if (e == cudaSuccess && (phases & 2)) e = dib_launch_reparam_bwd(a, d_emb, ldemb, beta_dev, inv_batch, d_out, st);
  return sync_result(fn, e, st);
}

// the compiled loss, its accuracy and d loss / d z of n rows, as the step's loss phase launches it (unit tests)
int dib_debug_loss(int32_t loss, int32_t out_act, float alpha, const float* pred, int32_t ldp, const float* y, int32_t out_dim,
                   int64_t n, float inv_batch, const float* weights, float* d_pred, float* user_pred, float* loss_part,
                   float* acc_part, int32_t round_out, void* stream) {
  const std::string fn = "dib_debug_loss: ";
  if (loss < DIB_LOSS_BCE_LOGITS || loss > DIB_LOSS_BCE_PROBS) return fail(fn + "unknown loss " + std::to_string(loss));
  if (out_act < DIB_ACT_LINEAR || out_act > DIB_ACT_ELU) return fail(fn + "unknown out_act " + std::to_string(out_act));
  if (out_dim < 1) return fail(fn + "needs out_dim >= 1");
  if (ldp < out_dim) return fail(fn + "needs ldp >= out_dim (ldp = " + std::to_string(ldp) + ")");
  if (n < 0 || n > 0x7fffffffll) return fail(fn + "needs 0 <= n < 2^31 (n = " + std::to_string(n) + ")");
  if (weights && loss == DIB_LOSS_EXTERNAL) return fail(fn + "the external loss takes no sample weights");
  if (!pred || !loss_part || !acc_part) return fail(fn + "pred, loss_part and acc_part must not be null");
  const cudaStream_t st = static_cast<cudaStream_t>(stream);
  const cudaError_t e = dib_launch_loss(loss, out_act, alpha, pred, ldp, y, out_dim, n, inv_batch, d_pred, user_pred, loss_part,
                                        acc_part, round_out ? 1 : 0, weights, st);
  return sync_result(fn, e, st);
}

// the header's C mirror of a reduction segment: the test hook hands its array to the launcher as it is
static_assert(sizeof(dib_reduce_seg) == sizeof(DibReduceSeg), "dib_reduce_seg size");
static_assert(offsetof(dib_reduce_seg, src) == offsetof(DibReduceSeg, src) &&
              offsetof(dib_reduce_seg, row_stride) == offsetof(DibReduceSeg, row_stride) &&
              offsetof(dib_reduce_seg, nrows) == offsetof(DibReduceSeg, nrows) &&
              offsetof(dib_reduce_seg, count) == offsetof(DibReduceSeg, count) &&
              offsetof(dib_reduce_seg, scale) == offsetof(DibReduceSeg, scale) &&
              offsetof(dib_reduce_seg, dst) == offsetof(DibReduceSeg, dst), "dib_reduce_seg layout");

// the step's fixed-order reductions: reduce_partials, reduce_segments or finalize_stats (unit tests)
int dib_debug_reduce(int32_t kind, const float* src, int64_t row_stride, int32_t nrows, int64_t count, float* dst,
                     const dib_reduce_seg* segs, int32_t nseg, const float* loss_part, const float* acc_part, int32_t nblk_loss,
                     int64_t n, int32_t has_y, void* stream) {
  const std::string fn = "dib_debug_reduce: ";
  auto shape_ok = [&](const std::string& what, int64_t rs, int64_t nr, int64_t cnt) -> bool {
    if (cnt < 0 || cnt > 0x7fffffffll || nr < 0 || (nr > 1 && rs < cnt)) {
      fail(fn + what + " needs 0 <= count < 2^31, nrows >= 0 and row_stride >= count (count = " + std::to_string(cnt) +
           ", nrows = " + std::to_string(nr) + ", row_stride = " + std::to_string(rs) + ")");
      return false;
    }
    return true;
  };
  const cudaStream_t st = static_cast<cudaStream_t>(stream);
  cudaError_t e;
  if (kind == 0) {
    if (!shape_ok("reduce_partials", row_stride, nrows, count)) return 1;
    if (count > 0 && (!src || !dst)) return fail(fn + "src and dst must not be null");
    e = dib_launch_reduce_partials(src, row_stride, nrows, count, dst, st);
  } else if (kind == 1) {
    if (nseg < 0 || (nseg > 0 && !segs)) return fail(fn + "needs nseg >= 0 segments");
    for (int s = 0; s < nseg; ++s) {
      if (segs[s].count <= 0) continue;
      if (!shape_ok("segment " + std::to_string(s), segs[s].row_stride, segs[s].nrows, segs[s].count)) return 1;
      if (!segs[s].src || !segs[s].dst) return fail(fn + "segment " + std::to_string(s) + ": src and dst must not be null");
    }
    e = dib_launch_reduce_segments(reinterpret_cast<const DibReduceSeg*>(segs), nseg, st);
  } else if (kind == 2) {
    if (nrows < 1) return fail(fn + "finalize_stats needs nrows = F >= 1");
    if (!shape_ok("finalize_stats", row_stride, nrows, count)) return 1;
    if (nblk_loss < 0 || n < 0) return fail(fn + "finalize_stats needs nblk_loss >= 0 and n >= 0");
    if (!src || !dst || (has_y && nblk_loss > 0 && (!loss_part || !acc_part)))
      return fail(fn + "finalize_stats needs src, dst and, with has_y, loss_part and acc_part");
    e = dib_launch_finalize_stats(src, (int)row_stride, (int)count, loss_part, acc_part, nblk_loss, nrows, n, has_y ? 1 : 0, dst, st);
  } else {
    return fail(fn + "kind is 0 (reduce_partials), 1 (reduce_segments) or 2 (finalize_stats)");
  }
  return sync_result(fn, e, st);
}

// the step's positional encoding (dib_launch_pe) with caller tables; the hook reads the tables to check them (unit tests)
int dib_debug_pe(const float* x, int32_t ldx, int32_t x_col_shift, const int32_t* col_src, const int32_t* col_freq,
                 int32_t col_begin, int32_t col_end, float* pe, int32_t ldpe, int32_t pe_col_shift, int64_t n,
                 const int32_t* row_index, const int32_t* col_feat, int64_t n_src, int32_t round_out, void* stream) {
  const std::string fn = "dib_debug_pe: ";
  if (col_begin < 0 || col_end < col_begin) return fail(fn + "needs 0 <= col_begin <= col_end");
  if (n < 0 || n > 0x7fffffffll) return fail(fn + "needs 0 <= n < 2^31 (n = " + std::to_string(n) + ")");
  if (!x || !col_src || !col_freq || !pe) return fail(fn + "x, col_src, col_freq and pe must not be null");
  if (row_index && (!col_feat || n_src < 1)) return fail(fn + "row_index needs col_feat and n_src >= 1");
  std::vector<int32_t> src(col_end), feat(row_index ? col_end : 0);
  if (col_end > 0) {
    DIB_CUDA_OK(cudaMemcpy(src.data(), col_src, col_end * sizeof(int32_t), cudaMemcpyDeviceToHost));
    if (row_index) DIB_CUDA_OK(cudaMemcpy(feat.data(), col_feat, col_end * sizeof(int32_t), cudaMemcpyDeviceToHost));
  }
  for (int c = col_begin; c < col_end; ++c) {
    if (c - pe_col_shift < 0 || c - pe_col_shift >= ldpe)
      return fail(fn + "column " + std::to_string(c) + " lands outside [0, ldpe) after pe_col_shift");
    if (src[c] >= 0 && (src[c] - x_col_shift < 0 || src[c] - x_col_shift >= ldx))
      return fail(fn + "col_src[" + std::to_string(c) + "] reads outside [0, ldx) after x_col_shift");
    if (row_index && src[c] >= 0 && feat[c] < 0) return fail(fn + "col_feat[" + std::to_string(c) + "] < 0");
  }
  const cudaStream_t st = static_cast<cudaStream_t>(stream);
  const cudaError_t e = dib_launch_pe(x, ldx, x_col_shift, col_src, col_freq, col_begin, col_end, pe, ldpe, pe_col_shift, n,
                                      round_out ? 1 : 0, st, row_index, col_feat, n_src);
  return sync_result(fn, e, st);
}

// the encoders' Keras Dropout, forward or backward in place, as the step launches it (unit tests)
int dib_debug_dropout(const float* src, float* dst, int64_t feat_stride, int32_t ld, int32_t width, int32_t F, int64_t n,
                      float rate, uint64_t seed, uint32_t step, const uint32_t* step_dev, uint64_t sample_offset, int32_t layer,
                      int32_t feature, int32_t backward, int32_t round_out, void* stream) {
  const std::string fn = "dib_debug_dropout: ";
  if (!(rate >= 0.f && rate < 1.f)) return fail(fn + "needs 0 <= rate < 1");
  if (width < 1 || ld < width) return fail(fn + "needs width >= 1 and ld >= width (width = " + std::to_string(width) + ")");
  if (F < 1 || F > 65535) return fail(fn + "needs 1 <= F <= 65535 (F = " + std::to_string(F) + ")");
  if (feature < -1 || feature >= F) return fail(fn + "needs -1 <= feature < F (feature = " + std::to_string(feature) + ")");
  if (layer < 0 || layer > 127) return fail(fn + "needs 0 <= layer < 128 (layer = " + std::to_string(layer) + ")");
  if (n < 0 || n > 0x7fffffffll) return fail(fn + "needs 0 <= n < 2^31 (n = " + std::to_string(n) + ")");
  if (feat_stride < n * ld) return fail(fn + "needs feat_stride >= n * ld");
  if (!dst || (!backward && !src)) return fail(fn + "needs dst, and src for the forward");
  const cudaStream_t st = static_cast<cudaStream_t>(stream);
  const cudaError_t e = dib_launch_dropout(backward ? nullptr : src, dst, feat_stride, ld, width, F, n, rate, seed, step, step_dev,
                                           sample_offset, layer, feature, backward ? 1 : 0, round_out ? 1 : 0, st);
  return sync_result(fn, e, st);
}

// the header's C mirror of a weight-gradient layer: the test hook hands its array to the launcher as it is
static_assert(sizeof(dib_int16_wgrad_layer) == sizeof(DibInt16Wgrad), "dib_int16_wgrad_layer size");
static_assert(offsetof(dib_int16_wgrad_layer, g_in) == offsetof(DibInt16Wgrad, g_in) &&
              offsetof(dib_int16_wgrad_layer, K) == offsetof(DibInt16Wgrad, K) &&
              offsetof(dib_int16_wgrad_layer, dz) == offsetof(DibInt16Wgrad, dz) &&
              offsetof(dib_int16_wgrad_layer, N) == offsetof(DibInt16Wgrad, N) &&
              offsetof(dib_int16_wgrad_layer, dW_part) == offsetof(DibInt16Wgrad, dW_part) &&
              offsetof(dib_int16_wgrad_layer, nsplit) == offsetof(DibInt16Wgrad, nsplit) &&
              offsetof(dib_int16_wgrad_layer, rows_per_split) == offsetof(DibInt16Wgrad, rows_per_split),
              "dib_int16_wgrad_layer layout");

// one dib_int16_fwd / dib_int16_dgrad / dib_int16_wgrad launch, as the 16-bit integration forward and backward issue them
// (unit tests)
int dib_debug_int16_gemm(int32_t mode, int32_t bf16, int32_t M, int32_t K, int32_t N, const void* a, int32_t lda,
                         const void* w16, const float* bias, const void* x, int32_t ldx, void* out, int32_t ldc, int32_t act,
                         float alpha, float* colsum, const dib_int16_wgrad_layer* layers, int32_t count, int64_t split_stride,
                         float out_scale, void* stream) {
  const std::string fn = "dib_debug_int16_gemm: ";
  if (mode < DIB_GEMM_FWD || mode > DIB_GEMM_WGRAD) return fail(fn + "unknown mode " + std::to_string(mode));
  if (bf16 != 0 && bf16 != 1) return fail(fn + "bf16 is 0 (fp16) or 1 (bf16)");
  if (M < 1) return fail(fn + "needs M >= 1 (M = " + std::to_string(M) + ")");
  const cudaStream_t st = static_cast<cudaStream_t>(stream);
  if (mode == DIB_GEMM_WGRAD) {
    if (count < 1 || count > 2 || !layers) return fail(fn + "WGRAD takes 1 or 2 layers (count = " + std::to_string(count) + ")");
    for (int q = 0; q < count; ++q) {
      const dib_int16_wgrad_layer& l = layers[q];
      const std::string lq = "layer " + std::to_string(q) + ": ";
      if (!dib_int16_gemm_ok(l.K, l.N))
        return fail(fn + lq + "needs K a positive multiple of 64 and N a positive multiple of 128 (K = " + std::to_string(l.K) +
                    ", N = " + std::to_string(l.N) + ")");
      if (!l.g_in || !l.dz || !l.dW_part) return fail(fn + lq + "g_in, dz and dW_part must not be null");
      DIB_HOOK_CHECK(int16_base_error("g_in", l.g_in));
      DIB_HOOK_CHECK(int16_base_error("dz", l.dz));
      if (reinterpret_cast<uintptr_t>(l.dW_part) % 8) return fail(fn + lq + "dW_part must be 8-byte aligned");
      if (l.nsplit < 1) return fail(fn + lq + "needs nsplit >= 1");
      if (l.rows_per_split < 64 || l.rows_per_split % 64)
        return fail(fn + lq + "needs rows_per_split a positive multiple of 64 (rows_per_split = " +
                    std::to_string(l.rows_per_split) + ")");
      const int64_t span = (int64_t)l.nsplit * l.rows_per_split;
      if (span < M) return fail(fn + lq + "needs nsplit * rows_per_split >= M (" + std::to_string(span) + " < " + std::to_string(M) + ")");
      if (span > 0x7fffffffll) return fail(fn + lq + "needs nsplit * rows_per_split < 2^31");
      if ((int64_t)l.K * l.N > split_stride || split_stride % 2)
        return fail(fn + lq + "every [K x N] partial slice must lie inside split_stride, an even count (split_stride = " +
                    std::to_string(split_stride) + ")");
    }
    return sync_result(fn, dib_int16_wgrad(reinterpret_cast<const DibInt16Wgrad*>(layers), count, M, split_stride, out_scale,
                                           bf16, st), st);
  }
  if (!dib_int16_gemm_ok(K, N))
    return fail(fn + "needs K a positive multiple of 64 and N a positive multiple of 128 (K = " + std::to_string(K) + ", N = " +
                std::to_string(N) + ")");
  if (!known_act(act)) return fail(fn + "unknown act " + std::to_string(act));
  if (!a || !w16 || !out) return fail(fn + "a, w16 and out must not be null");
  const int in_w = mode == DIB_GEMM_FWD ? K : N, out_w = mode == DIB_GEMM_FWD ? N : K;
  DIB_HOOK_CHECK(int16_base_error("a", a));
  DIB_HOOK_CHECK(int16_base_error("w16", w16));
  DIB_HOOK_CHECK(int16_base_error("out", out));
  DIB_HOOK_CHECK(int16_ld_error("lda", lda, in_w));
  DIB_HOOK_CHECK(int16_ld_error("ldc", ldc, out_w));
  if (mode == DIB_GEMM_FWD) {
    if (!bias) return fail(fn + "FWD needs bias");
    DIB_HOOK_CHECK(int16_bias_error("bias", bias));
    return sync_result(fn, dib_int16_fwd(a, lda, w16, bias, out, ldc, M, K, N, act, alpha, bf16, st), st);
  }
  if (x) {
    DIB_HOOK_CHECK(int16_base_error("x", x));
    DIB_HOOK_CHECK(int16_ld_error("ldx", ldx, K));
  }
  return sync_result(fn, dib_int16_dgrad(a, lda, w16, x, ldx, out, ldc, M, K, N, act, alpha, colsum, bf16, st), st);
}

// the output head of the 16-bit integration network, generic or out = 1, as the step's forward launches it (unit tests)
int dib_debug_int16_head(int32_t head1, int32_t bf16, const void* g, int32_t ldg, int32_t K, const float* Wc, const float* bc,
                         int32_t out_dim, int32_t out_act, int32_t hid_act, float alpha, int32_t loss, const float* y, int64_t n,
                         float inv_batch, float gscale, void* dg, int32_t lddg, float* user_pred, float* wpart,
                         int32_t wpart_stride, float* loss_part, float* acc_part, int32_t nblocks, const float* weights,
                         void* stream) {
  const std::string fn = "dib_debug_int16_head: ";
  if (head1 != 0 && head1 != 1) return fail(fn + "head1 is 0 (generic kernel) or 1 (the out = 1 kernel)");
  if (bf16 != 0 && bf16 != 1) return fail(fn + "bf16 is 0 (fp16) or 1 (bf16)");
  if (!dib_int16_head_ok(K, out_dim, head1 != 0))
    return fail(fn + "needs K == 256 and 1 <= out_dim <= 16, and head1 needs out_dim == 1 (K = " + std::to_string(K) +
                ", out_dim = " + std::to_string(out_dim) + ", head1 = " + std::to_string(head1) + ")");
  if (!known_act(out_act) || !known_act(hid_act)) return fail(fn + "unknown out_act or hid_act");
  if (loss < DIB_LOSS_BCE_LOGITS || loss > DIB_LOSS_BCE_PROBS || loss == DIB_LOSS_EXTERNAL)
    return fail(fn + "unknown loss " + std::to_string(loss) + " (the head computes bce_logits, sparse CE, mse or bce_probs)");
  if (n < 1 || n > 0x7fffffffll) return fail(fn + "needs 1 <= n < 2^31 (n = " + std::to_string(n) + ")");
  if (nblocks < 1 || nblocks > 65535) return fail(fn + "needs 1 <= nblocks <= 65535 (nblocks = " + std::to_string(nblocks) + ")");
  if (!g || !Wc || !bc || !loss_part || !acc_part) return fail(fn + "g, Wc, bc, loss_part and acc_part must not be null");
  DIB_HOOK_CHECK(int16_base_error("g", g));
  DIB_HOOK_CHECK(int16_ld_error("ldg", ldg, K));
  if (weights && !y) return fail(fn + "weights need y");
  if (dg) {
    DIB_HOOK_CHECK(int16_base_error("dg", dg));
    DIB_HOOK_CHECK(int16_ld_error("lddg", lddg, K));
    if (!wpart) return fail(fn + "training (dg) needs wpart");
    if (wpart_stride < K * out_dim + out_dim + K)
      return fail(fn + "needs wpart_stride >= K * out_dim + out_dim + K (wpart_stride = " + std::to_string(wpart_stride) + ")");
  }
  const cudaStream_t st = static_cast<cudaStream_t>(stream);
  return sync_result(fn, dib_int16_head(g, ldg, K, Wc, bc, out_dim, out_act, hid_act, alpha, loss, y, n, inv_batch, gscale, dg,
                                        lddg, user_pred, wpart, wpart_stride, loss_part, acc_part, nblocks, head1 != 0, weights,
                                        bf16, st), st);
}

// the fused integration tail, forward only, with the training head, or with its dgrad stages, as the step's forward launches
// it (unit tests)
int dib_debug_int16_fwd2(int32_t bf16, const void* g_in, int32_t ld_in, int32_t K0, const void* w16_0, const float* b0,
                         const void* w16_1, const float* b1, void* g1, const float* wout, const float* bout, int32_t act,
                         int32_t out_act, float alpha, int32_t loss, const float* y, int32_t M, float inv_batch, float gscale,
                         void* dg2, void* dg1, float* dbpart, void* demb, float* user_pred, float* wpart, int32_t wpart_stride,
                         float* loss_part, float* acc_part, const float* weights, int32_t* nblocks, void* stream) {
  const std::string fn = "dib_debug_int16_fwd2: ";
  if (bf16 != 0 && bf16 != 1) return fail(fn + "bf16 is 0 (fp16) or 1 (bf16)");
  if (!dib_int16_fwd2_ok(K0, 256, 256, 1)) return fail(fn + "needs K0 a positive multiple of 64 (K0 = " + std::to_string(K0) + ")");
  if (M < 1) return fail(fn + "needs M >= 1 (M = " + std::to_string(M) + ")");
  if (!known_act(act) || !known_act(out_act)) return fail(fn + "unknown act or out_act");
  if (loss < DIB_LOSS_BCE_LOGITS || loss > DIB_LOSS_BCE_PROBS || loss == DIB_LOSS_EXTERNAL)
    return fail(fn + "unknown loss " + std::to_string(loss) + " (the tail computes bce_logits, sparse CE, mse or bce_probs)");
  if (!g_in || !w16_0 || !b0 || !w16_1 || !b1 || !g1 || !wout || !bout || !loss_part || !acc_part || !nblocks)
    return fail(fn + "g_in, w16_0, b0, w16_1, b1, g1, wout, bout, loss_part, acc_part and nblocks must not be null");
  DIB_HOOK_CHECK(int16_base_error("g_in", g_in));
  DIB_HOOK_CHECK(int16_ld_error("ld_in", ld_in, K0));
  DIB_HOOK_CHECK(int16_base_error("w16_0", w16_0));
  DIB_HOOK_CHECK(int16_base_error("w16_1", w16_1));
  DIB_HOOK_CHECK(int16_base_error("g1", g1));
  DIB_HOOK_CHECK(int16_base_error("dg2", dg2));
  DIB_HOOK_CHECK(int16_base_error("dg1", dg1));
  DIB_HOOK_CHECK(int16_base_error("demb", demb));
  if (reinterpret_cast<uintptr_t>(b0) % 16 || reinterpret_cast<uintptr_t>(b1) % 16 || reinterpret_cast<uintptr_t>(wout) % 16)
    return fail(fn + "b0, b1 and wout must be 16-byte aligned");
  if (weights && !y) return fail(fn + "weights need y");
  if (dg1 && (!dg2 || !dbpart)) return fail(fn + "dg1 needs dg2 and dbpart");
  if (demb && !dg1) return fail(fn + "demb needs dg1");
  if (dg2 && !wpart) return fail(fn + "training (dg2) needs wpart");
  if (dg2 && wpart_stride < 256 + 1 + 256)
    return fail(fn + "needs wpart_stride >= 513 (wpart_stride = " + std::to_string(wpart_stride) + ")");
  const cudaStream_t st = static_cast<cudaStream_t>(stream);
  return sync_result(fn, dib_int16_fwd2_head(g_in, ld_in, K0, w16_0, b0, w16_1, b1, g1, wout, bout, act, out_act, alpha, loss, y,
                                             M, inv_batch, gscale, dg2, dg1, dbpart, demb, user_pred, wpart, wpart_stride,
                                             loss_part, acc_part, nblocks, weights, bf16, st), st);
}

// the fused encoder kernels (dib_enc_fused.cu): the weight pack, the forward and the backward, as forward_encoders and
// backward_encoders launch them, on a grid the caller picks (unit tests)
int dib_debug_enc_fused(int32_t phases, int32_t F, const int32_t* fdim, const int32_t* x_off, int32_t nfreq, int32_t act,
                        float alpha, int32_t bf16, float logvar_offset, const float* params, int64_t param_count,
                        const int64_t* w0_off, const int64_t* b0_off, const int64_t* w1_off, const int64_t* b1_off,
                        const int64_t* w2_off, const int64_t* b2_off, int32_t grid, int64_t n, const float* x, int32_t ldx,
                        const float* eps, uint64_t seed, uint32_t step, const uint32_t* step_dev, uint64_t sample_offset,
                        float* emb, int32_t ldemb, float* user_emb, void* emb16, int32_t ldemb16, float* kl_part,
                        int32_t kl_stride, const float* d_emb, int32_t ldd, const void* d_emb16, int32_t ldd16,
                        const float* beta_dev, float inv_batch, float gscale, float* part, int64_t split_stride, void* packed,
                        void* stream) {
  const std::string fn = "dib_debug_enc_fused: ";
  auto str = [](long long v) { return std::to_string(v); };
  auto misaligned = [](const void* p, uintptr_t a) { return reinterpret_cast<uintptr_t>(p) % a != 0; };
  if (phases < 1 || phases > 7) return fail(fn + "phases is a mask of 1 (pack), 2 (forward) and 4 (backward) (phases = " + str(phases) + ")");
  if (F < 1 || F > 65535) return fail(fn + "needs 1 <= F <= 65535 (F = " + str(F) + ")");
  if (!fdim || !x_off) return fail(fn + "fdim and x_off must not be null");
  if (nfreq < 1) return fail(fn + "needs nfreq >= 1 (nfreq = " + str(nfreq) + ")");
  if (!known_act(act)) return fail(fn + "unknown act " + str(act));
  if (bf16 != 0 && bf16 != 1) return fail(fn + "bf16 is 0 (fp16) or 1 (bf16)");
  if (!w0_off || !b0_off || !w1_off || !b1_off || !w2_off || !b2_off) return fail(fn + "the six offset tables must not be null");
  if (!params || param_count < 1) return fail(fn + "needs params and param_count >= 1");
  if (!packed || misaligned(packed, 16)) return fail(fn + "packed must be a 16-byte aligned buffer of the 16-bit image");
  const bool fwd = phases & 2, bwd = phases & 4;
  // every feature's x columns and parameter blocks (w_in = fdim nfreq first-layer inputs, hidden 128, 2E = 64 outputs)
  const int64_t span = bwd ? std::min<int64_t>(param_count, split_stride) : param_count;
  for (int f = 0; f < F; ++f) {
    const std::string at = " of feature " + str(f);
    if (!dib_enc_fused_feature_ok(fdim[f], nfreq))
      return fail(fn + "needs 1 <= fdim <= 3 and fdim nfreq + 1 <= 16 (fdim" + at + " = " + str(fdim[f]) + ", nfreq = " +
                  str(nfreq) + ")");
    if ((fwd || bwd) && (x_off[f] < 0 || (int64_t)x_off[f] + fdim[f] > ldx))
      return fail(fn + "the x columns" + at + " must lie inside [0, ldx) (x_off = " + str(x_off[f]) + ", ldx = " + str(ldx) + ")");
    const int64_t off[6] = {w0_off[f], b0_off[f], w1_off[f], b1_off[f], w2_off[f], b2_off[f]};
    const int64_t size[6] = {(int64_t)fdim[f] * nfreq * 128, 128, 128 * 128, 128, 128 * 64, 64};
    static const char* names[6] = {"w0_off", "b0_off", "w1_off", "b1_off", "w2_off", "b2_off"};
    for (int k = 0; k < 6; ++k)
      if (off[k] < 0 || off[k] + size[k] > span)
        return fail(fn + "the parameter block " + names[k] + at + " must lie inside params" + (bwd ? " and split_stride" : "") +
                    " (offset " + str(off[k]) + ", size " + str(size[k]) + ")");
    if (bwd && (w1_off[f] % 2 || w2_off[f] % 2)) return fail(fn + "w1_off and w2_off" + at + " must be even (float2 stores)");
  }
  const cudaStream_t st = static_cast<cudaStream_t>(stream);
  const long long tiles = (n + 127) / 128, want = (long long)F * tiles;
  if ((fwd || bwd) && (n < 1 || n > 0x7fffffffll)) return fail(fn + "needs 1 <= n < 2^31 (n = " + str(n) + ")");
  int sms = 0, dev = 0;
  if (cudaGetDevice(&dev) != cudaSuccess || cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess)
    return fail(fn + "cannot read the multiprocessor count");
  // grid 0: the library's choice for the phase (forward: two CTAs per SM, backward: one)
  const long long cap_fwd = (long long)sms * dib_enc_fused_fwd_ctas_per_sm(), cap_bwd = sms;
  const int grid_fwd = grid ? grid : (int)std::min(want, cap_fwd), grid_bwd = grid ? grid : (int)std::min(want, cap_bwd);
  if ((fwd || bwd) && (grid < 0 || grid > want))
    return fail(fn + "needs 0 <= grid <= F ceil(n / 128) = " + str(want) + " (grid = " + str(grid) + ")");
  if (fwd) {
    if (!x) return fail(fn + "the forward needs x");
    if (!emb && !emb16 && !user_emb) return fail(fn + "the forward needs emb, user_emb or emb16");
    if (emb && (misaligned(emb, 8) || ldemb % 2 || ldemb < F * 32))
      return fail(fn + "emb must be 8-byte aligned with ldemb even and >= F * 32 (ldemb = " + str(ldemb) + ")");
    if (user_emb && misaligned(user_emb, 8)) return fail(fn + "user_emb must be 8-byte aligned");
    if (emb16 && (misaligned(emb16, 4) || ldemb16 % 2 || ldemb16 < F * 32))
      return fail(fn + "emb16 must be 4-byte aligned with ldemb16 even and >= F * 32 (ldemb16 = " + str(ldemb16) + ")");
    if (!kl_part) return fail(fn + "the forward needs kl_part");
    if (kl_stride < (grid_fwd + F - 1) / F)
      return fail(fn + "needs kl_stride >= ceil(grid / F) = " + str((grid_fwd + F - 1) / F) + " (kl_stride = " + str(kl_stride) + ")");
  }
  if (bwd) {
    if (!x) return fail(fn + "the backward needs x");
    if (!d_emb == !d_emb16) return fail(fn + "the backward takes exactly one of d_emb and d_emb16");
    if (d_emb && (misaligned(d_emb, 8) || ldd % 2 || ldd < F * 32))
      return fail(fn + "d_emb must be 8-byte aligned with ldd even and >= F * 32 (ldd = " + str(ldd) + ")");
    if (d_emb16 && (misaligned(d_emb16, 16) || ldd16 % 8 || ldd16 < F * 32))
      return fail(fn + "d_emb16 must be 16-byte aligned with ldd16 a multiple of 8 and >= F * 32 (ldd16 = " + str(ldd16) + ")");
    if (!beta_dev) return fail(fn + "the backward needs beta_dev");
    int ex = 0;
    if (!(gscale > 0.f) || std::isinf(gscale) || std::frexp(gscale, &ex) != 0.5f)
      return fail(fn + "gscale must be a power of two (gscale = " + std::to_string(gscale) + ")");
    if (!part || misaligned(part, 8) || split_stride % 2)
      return fail(fn + "the backward needs part 8-byte aligned and split_stride even (split_stride = " + str(split_stride) + ")");
  }
  if (eps && misaligned(eps, 8)) return fail(fn + "eps must be 8-byte aligned");
  // the descriptor tables live on the device, as dib_create leaves them
  DibEncFusedDesc d;
  d.F = F; d.nfreq = nfreq; d.act = act; d.alpha = alpha; d.bf16 = bf16; d.logvar_offset = logvar_offset;
  const int64_t* off[6] = {w0_off, b0_off, w1_off, b1_off, w2_off, b2_off};
  void* dt = nullptr;
  DIB_CUDA_OK(dib_enc_fused_upload_tables(d, off, x_off, fdim, &dt));
  DibEncFusedIO io;
  io.params = params; io.packed = packed; io.x = x; io.ldx = ldx; io.n = n;
  io.eps = eps; io.seed = seed; io.step = step; io.step_dev = step_dev; io.sample_offset = sample_offset;
  io.emb = nullptr; io.ldemb = 0; io.user_emb = nullptr; io.kl_part = nullptr; io.kl_stride = 0;
  cudaError_t e = cudaSuccess;
  if (phases & 1) {
    // the pack kernel also clears the KL partial table when it fits its grid, as forward_encoders has it do
    const long long zn = kl_part ? (long long)F * kl_stride : 0;
    const bool clear = zn > 0 && zn <= dib_enc_fused_pack_zero_capacity(F);
    e = dib_enc_fused_pack(d, params, packed, clear ? kl_part : nullptr, clear ? zn : 0, st);
  }
  if (e == cudaSuccess && fwd) {
    DibEncFusedIO fo = io;
    fo.emb = emb; fo.ldemb = ldemb; fo.user_emb = user_emb; fo.kl_part = kl_part; fo.kl_stride = kl_stride;
    fo.emb16 = emb16; fo.ldemb16 = ldemb16;
    d.grid = grid_fwd;
    e = dib_enc_fused_forward(d, fo, st);
  }
  if (e == cudaSuccess && bwd) {
    DibEncFusedBwdIO b;
    b.d_emb = d_emb; b.ldd = ldd; b.d_emb16 = d_emb16; b.ldd16 = d_emb16 ? ldd16 : 0;
    b.beta_dev = beta_dev; b.inv_batch = inv_batch; b.gscale = gscale; b.part = part; b.split_stride = split_stride;
    d.grid = grid_bwd;
    e = dib_enc_fused_backward(d, io, b, st);
  }
  const int r = sync_result(fn, e, st);
  cudaFree(dt);
  return r;
}

}  // extern "C"
