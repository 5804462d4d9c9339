// dib_kernels.h -- internal launcher prototypes shared by the translation units of libdib_b200.so.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include <string>

struct DibGemmProblem;

// number of kernels launched by this library in this process (bench.py reports it as gpu_launches)
void dib_note_launch(int n = 1);

// records msg as this thread's dib_last_error() and returns 1, the C ABI's error code (dib_api.cu)
int fail(const std::string& msg);

#define DIB_CUDA_OK(expr)                                                                        \
  do {                                                                                           \
    cudaError_t _e = (expr);                                                                     \
    if (_e != cudaSuccess)                                                                       \
      return fail(std::string(#expr) + ": " + cudaGetErrorString(_e));                           \
  } while (0)

struct DibGemmLaunch {
  const DibGemmProblem* probs;  // device array, nprob entries
  int nprob;
  const float* baseA;
  const float* baseB;
  float* baseC;
  float* baseX;
  int M;               // batch rows
  int maxC, maxR;      // largest C (and, for WGRAD, R) over the group -> grid size
  int nsplit;          // WGRAD batch splits
  int rows_per_split;
  long long split_stride;
  float alpha;
  int round_out = 0;              // round FWD / DGRAD outputs to the TF32 grid (tensor-core mode operands)
  const float* baseBias = nullptr; // FWD bias base when baseB points at the TF32-rounded weight shadow
};

// problems per launch of a group whose every problem takes `z_per_problem` grid slices along z (WGRAD: nsplit, else 1):
// gridDim.z is at most 65 535, so larger groups run as several launches of this many problems (0: one problem does not fit)
inline int dib_gemm_chunk_problems(int nprob, int z_per_problem) {
  const int cap = 65535 / (z_per_problem > 0 ? z_per_problem : 1);
  return nprob < cap ? nprob : cap;
}

cudaError_t dib_launch_gemm_simt(int mode, const DibGemmLaunch& L, cudaStream_t st);

// TF32 wgmma path (dib_gemm_tc.cu); `hp` = host copies of the group's problem descriptors
bool dib_gemm_tc_eligible(int mode, const DibGemmProblem* hp, int nprob, const float* params_base_hint);
cudaError_t dib_launch_gemm_tc(int mode, const DibGemmLaunch& L, const DibGemmProblem* hp, cudaStream_t st);

// ---- elementwise / reduction kernels (dib_elementwise.cu) -----------------------------------------------
// positional encoding (models.py:22-23) into the padded first-layer operand; tables are per pe column.
cudaError_t dib_launch_pe(const float* x, int ldx, int x_col_shift, const int* col_src, const int* col_freq,
                          int col_begin, int col_end, float* pe, int ldpe, int pe_col_shift, int64_t n,
                          int round_out, cudaStream_t st, const int* row_index = nullptr,
                          const int* col_feat = nullptr, int64_t n_src = 0);

struct DibReparamArgs {
  const float* enc_out;    // [F][feat_stride] rows of ldo floats: (mu[E] | logvar[E] | pad)
  long long feat_stride;
  int ldo;
  const float* eps;        // [n, F, E] or nullptr -> Philox
  uint64_t seed; uint32_t step; uint64_t sample_offset;
  const uint32_t* step_dev = nullptr;   // optional device addend of `step` (CUDA-Graph replay)
  int F, E;
  int64_t n;
  int round_out = 0;
  // variable set sizes: rows are sets of set_len padded particle rows, set s has set_sizes[s] real ones; a padding row gets
  // u = 0, no KL and d(mu, logvar) = 0 (set_sizes[s] clamped into [1, set_len], dib_set_len).  nullptr: every row is real
  const int* set_sizes = nullptr; int set_len = 1;
};
// u = mu + exp(logvar/2) eps (models.py:108); per-(block,feature) partial sums of the KL (models.py:111-112).
cudaError_t dib_launch_reparam_fwd(const DibReparamArgs& a, float* emb, int ldemb, float* user_emb,
                                   float* kl_part, int nblk_stride, cudaStream_t st);
// d(mu,logvar) from d(u) and beta * dKL (models.py:118).
cudaError_t dib_launch_reparam_bwd(const DibReparamArgs& a, const float* d_emb, int ldemb, const float* beta_dev,
                                   float inv_batch, float* d_out, cudaStream_t st);

// compiled loss + metrics=['accuracy'] + d(loss)/d(pre-activation output); weights: the n rows' sample weights or null.
cudaError_t dib_launch_loss(int loss, int out_act, float alpha, const float* pred, int ldp, const float* y, int out_dim,
                            int64_t n, float inv_batch, float* d_pred /*nullable*/, float* user_pred /*nullable*/,
                            float* loss_part, float* acc_part, int round_out, const float* weights /*nullable*/, cudaStream_t st);
// Keras' class_weight map of n rows: out[i] = table[class of y row i] (* sw[i]); see dib_class_weight_rows
cudaError_t dib_launch_class_weight_rows(const float* y, int64_t n, int y_cols, const float* table, int classes, const float* sw,
                                         float* out, cudaStream_t st);

// ---- compiled metrics (dib_metrics.cu; dib_set_metrics) -----------------------------------------------------------
constexpr int kDibMaxMetrics = 16;                 // DIB_MAX_METRICS
constexpr int kDibMetricMaxCtas = 128;             // CTA partials in the workspace: kDibMetricMaxCtas * tail floats
struct DibMetricTable {
  int count = 0;                                   // metrics
  int tail = 0;                                    // floats of the metric tail
  int buckets = 0;                                 // sum over the confusion metrics of (T + 1)
  bool sigmoid = false;                            // some confusion metric reads sigmoid(z)
  int kind[kDibMaxMetrics], weighted[kDibMaxMetrics], from_logits[kDibMaxMetrics], nthr[kDibMaxMetrics];
  int off[kDibMaxMetrics];                         // first tail float of metric k
  int boff[kDibMaxMetrics];                        // confusion: first entry of its threshold table / bucket row
  float threshold[kDibMaxMetrics];
};
// z [n, out_dim] and y ([n] labels or [n, out_dim]) -> tail [t.tail]; w: the rows' sample weights or null; part: the
// workspace's CTA partials, counter: a zeroed device word the last CTA resets
cudaError_t dib_launch_metrics(const DibMetricTable& t, const float* z, const float* y, int out_dim, int64_t n, const float* w,
                               float* part, unsigned int* counter, float* tail, cudaStream_t st);
// host-side set-up of a table's launches (the shared-memory opt-in); call before the first launch and outside graph capture
cudaError_t dib_metrics_prepare(const DibMetricTable& t);
cudaError_t dib_launch_metrics_update_tail(const float* tail, double* acc, int count, cudaStream_t st);

cudaError_t dib_launch_round_copy(const float* src, float* dst, int64_t count, cudaStream_t st);

cudaError_t dib_launch_finalize_stats(const float* kl_part, int nblk_stride, int nblk_kl, const float* loss_part,
                                      const float* acc_part, int nblk_loss, int F, int64_t n, int has_y,
                                      float* out_stats, cudaStream_t st);

cudaError_t dib_launch_reduce_partials(const float* part, long long split_stride, int nsplit, int64_t count,
                                       float* out, cudaStream_t st);

cudaError_t dib_launch_copy2d(const float* src, int lds, float* dst, int ldd, int cols, int64_t n, cudaStream_t st);

cudaError_t dib_launch_optimizer(int kind, float* params, const float* grads, float* s1, float* s2, int64_t count,
                                 const float* lr_dev, int32_t* step_dev, float h0, float h1, float h2, cudaStream_t st);
cudaError_t dib_launch_pe_plain(const float* x, int64_t n, int d, int nfreq, float* out, cudaStream_t st);

cudaError_t dib_launch_adam(float* params, const float* grads, float* m, float* v, int64_t count,
                            const float* lr_dev, int32_t* step_dev, float b1, float b2, float eps, cudaStream_t st);

// mode 0: Bhattacharyya distance, 1: KL(1||2); ml* rows are (mu[E] | logvar[E]) with leading dimension ld*, `groups`
// independent problems gstride* floats apart; outputs [groups, n, m].
cudaError_t dib_launch_pairwise_gauss(int mode, const float* ml1, int64_t ld1, int64_t gstride1, int64_t n,
                                      const float* ml2, int64_t ld2, int64_t gstride2, int64_t m, int E, int groups,
                                      float* out_dist, float* out_comp, cudaStream_t st);

// next row f3 (dib_infonce.cu): kind 0 l2sq | 1 l2 | 2 l1 | 3 linf | 4 cosine
cudaError_t dib_launch_similarity(int kind, const float* e1, int64_t n, const float* e2, int64_t m, int d, float temperature,
                                  float* out, cudaStream_t st);
cudaError_t dib_launch_infonce_head(int kind, const float* e1, const float* e2, int64_t n, int d, float temperature,
                                    float* scratch, float* out_loss, float* d_e1, float* d_e2, cudaStream_t st);

// the InfoNCE loss of DIB_LOSS_INFONCE with memory linear in n (dib_infonce_stream.cu): e1 [n, d] (ld1), e2 [n, d] (ld2), d <= 512.
// The sweeps cover the own rows [row0, row0 + rows) of both sides against all n rows of the other side (one rank of a
// data-parallel group; row0 = 0, rows = n on one GPU).  Every index below is global unless it says otherwise.
struct DibInfonceStream {
  int kind; float temperature;
  const float* e1; int ld1;
  const float* e2; int ld2;
  int64_t n; int d;
  int64_t row0, rows;
  float* lse_r;                    // row log-sum-exps r_i at lse_r[i * lse_stride]: written for own i, read for all i
  float* lse_c;                    // column log-sum-exps c_j at lse_c[j * lse_stride]: likewise
  int lse_stride;
  float* diag;                     // [rows] s_ii of the own rows, local index
  float* loss_sum;                 // [1] = sum_{own i} (r_i + c_i - 2 s_ii) (= n * loss on one GPU)
  float* acc_zero;                 // [1] = 0 (the accuracy slot of the stats), nullable
  float* d_e1; int ld_d1;          // d loss / d e1, d loss / d e2 of the own rows at local index (pad columns zeroed); each
  float* d_e2; int ld_d2;          // nullable
  int round_out;                   // round the gradients to the TF32 grid (tensor-core operands)
};
// the row / column sweeps and the loss; then (after it, reading r and c of all n rows) the two gradient sweeps
cudaError_t dib_launch_infonce_stream_loss(const DibInfonceStream& a, cudaStream_t st);
cudaError_t dib_launch_infonce_stream_grads(const DibInfonceStream& a, cudaStream_t st);

cudaError_t dib_launch_metrics_update(const float* stats, const float* beta_dev, float* acc, int F, float kl_exponent,
                                      float kl_scale, cudaStream_t st);

// ---- custom-step variants (SURVEY 8f3) ----
// enc_out[f][row][E + e] += offset  (nb-particle cell 8: logvar offset), all features or only `feature` (>= 0)
cudaError_t dib_launch_add_logvar_offset(float* enc_out, long long feat_stride, int ldo, int F, int E, int64_t n, float offset,
                                         int feature, cudaStream_t st);
// nb-bool cell 4 SimpleEncoder forward: enc_out[f][row] = (x[row, x_off[f] + e] * mu_scaling_f | logvar_f), e < E
cudaError_t dib_launch_simple_enc_fwd(const float* x, int ldx, const int* x_off_dev, const float* params, float* enc_out,
                                      long long feat_stride, int ldo, int F, int E, int64_t n, int feature, int x_is_feature_only,
                                      const int* row_index, int64_t n_src, cudaStream_t st);
// its weight gradients: part[split][2f] = sum_rows sum_e d_mu * x, part[split][2f+1] = sum_rows sum_e d_logvar
cudaError_t dib_launch_simple_enc_wgrad(const float* x, int ldx, const int* x_off_dev, const float* d_out, long long feat_stride,
                                        int ldo, int F, int E, int64_t n, int nsplit, int rows_per_split, float* part,
                                        long long split_stride, cudaStream_t st);
// Keras Dropout on the encoder activations [F][feat_stride] rows of ld floats, `width` live columns (nb-radial cell 5):
//   backward == 0: dst = src * keep / (1 - rate)   (rate == 0: plain copy -- inference, where Dropout is the identity)
//   backward == 1: dst *= keep / (1 - rate)         (src ignored)
// keep from Philox (seed, step [+ *step_dev], sample_offset + row, feature, layer, column): oracle/philox.py :: dropout_keep
cudaError_t dib_launch_dropout(const float* src, float* dst, long long feat_stride, int ld, int width, int F, int64_t n, float rate,
                               uint64_t seed, uint32_t step, const uint32_t* step_dev, uint64_t sample_offset, int layer,
                               int feature, int backward, int round_out, cudaStream_t st);

// beta_eff = beta * scale * p * (sum_i stats[i] * inv_global_batch)^(p-1)   (d(beta*scale*KL^p)/dKL; p = 1: beta * scale)
cudaError_t dib_launch_beta_eff(const float* stats, int F, float inv_global_batch, const float* beta_dev, float exponent,
                                float scale, float* beta_eff_dev, cudaStream_t st);

// ---- fused per-feature encoder kernels (dib_enc_fused.cu): x -> emb / KL without touching HBM in between ----
struct DibEncFusedDesc {        // static per model; all pointers are DEVICE arrays of length F
  int F = 0, nfreq = 1, act = 0, bf16 = 0, grid = 0;
  float alpha = 0.2f;
  float logvar_offset = 0.f;      // folded into the logvar half of the b2 bias carrier when the weights are packed
  const int* x_off = nullptr; const int* fdim = nullptr;
  const long long* w0_off = nullptr; const long long* b0_off = nullptr; const long long* w1_off = nullptr;
  const long long* b1_off = nullptr; const long long* w2_off = nullptr; const long long* b2_off = nullptr;
};
struct DibEncFusedIO {
  const float* params; const void* packed;      // fp32 masters, packed 16-bit weights (dib_enc_fused_pack)
  const float* x; int ldx; int64_t n;
  const float* eps; uint64_t seed; uint32_t step; uint64_t sample_offset;
  const uint32_t* step_dev = nullptr;       // optional device addend of `step` (CUDA-Graph replay)
  float* emb; int ldemb; float* user_emb;
  float* kl_part; int kl_stride;
  void* emb16 = nullptr; int ldemb16 = 0;   // optional fp16 copy of emb (16-bit integration path)
};
// the shapes the fused encoder kernels run; the descriptor tables (off[k][f]: offset k of w0, b0, w1, b1, w2, b2 of feature
// f < d.F; x_off, fdim) copied to one device allocation *tables (the caller frees it) that d's table pointers point into
bool dib_enc_fused_shape_ok(int layers, const int* hidden, int E);
bool dib_enc_fused_feature_ok(int fdim, int nfreq);
cudaError_t dib_enc_fused_upload_tables(DibEncFusedDesc& d, const int64_t* const off[6], const int* x_off, const int* fdim,
                                        void** tables);
size_t dib_enc_fused_pack_bytes(int F);
long long dib_enc_fused_pack_zero_capacity(int F);
int dib_enc_fused_fwd_ctas_per_sm();
cudaError_t dib_enc_fused_pack(const DibEncFusedDesc& d, const float* params, void* packed, float* zero, long long zero_n, cudaStream_t st);
cudaError_t dib_enc_fused_forward(const DibEncFusedDesc& d, const DibEncFusedIO& io, cudaStream_t st);

struct DibEncFusedBwdIO {
  const float* d_emb; int ldd;          // gradient w.r.t. emb (scaled by 1/B_global), or null when d_emb16 is given
  const void* d_emb16 = nullptr; int ldd16 = 0;   // fp16 gradient already multiplied by gscale
  const float* beta_dev; float inv_batch; float gscale;
  float* part; long long split_stride;  // [slot][P] weight-gradient partials
};
cudaError_t dib_enc_fused_backward(const DibEncFusedDesc& d, const DibEncFusedIO& io, const DibEncFusedBwdIO& b,
                                   cudaStream_t st);

// ---- 16-bit integration network path (dib_int16.cu) ----
cudaError_t dib_int16_convert_many(const float* const* src, void* const* dst16, const long long* n, int count, int bf16, cudaStream_t st);
cudaError_t dib_int16_fwd(const void* g_in, int ld_in, const void* w16, const float* bias, void* g_out, int ld_out, int M,
                          int K, int N, int act, float alpha, int bf16, cudaStream_t st);
// colsum_part (nullable): [ceil(M/128)][K] per-row-tile column sums of dz_in = bias-gradient partials of the layer below
cudaError_t dib_int16_dgrad(const void* dz, int ld_dz, const void* w16, const void* g_in, int ld_g, void* dz_in, int ld_out,
                            int M, int K, int N, int act, float alpha, float* colsum_part, int bf16, cudaStream_t st);
// several column-sum reductions in ONE launch: dst[i] = scale * sum_{r < nrows} src[r * row_stride + i], i < count (fixed order)
struct DibReduceSeg { const float* src; long long row_stride; int nrows; long long count; float scale; float* dst; };
constexpr int kDibMaxReduceSegs = 8;
cudaError_t dib_launch_reduce_segments(const DibReduceSeg* segs, int nseg, cudaStream_t st);
// one layer's weight gradient: fp32 split partials of dW[K x N] = g_in[M x K]^T dz[M x N] (leading dimensions K and N) over
// nsplit batch slices of rows_per_split rows
struct DibInt16Wgrad { const void* g_in; int K; const void* dz; int N; float* dW_part; int nsplit; int rows_per_split; };
// the weight gradients of one or two layers (count = 1 or 2) in one launch, same batch M and partial stride
cudaError_t dib_int16_wgrad(const DibInt16Wgrad* layers, int count, int M, long long split_stride, float out_scale, int bf16,
                            cudaStream_t st);
int dib_int16_head_blocks(int num_sms);
// widths the 16-bit GEMMs run (a layer of fan-in K, fan-out N) and the output head runs (hidden width K; head1: out = 1 kernel)
bool dib_int16_gemm_ok(int K, int N);
bool dib_int16_head_ok(int K, int out_dim, bool head1);
// shapes the fused tail kernel (dib_int16_fwd2_head) handles: fan-in K0 of its first layer, its two widths, the output width
bool dib_int16_fwd2_ok(int K0, int N1, int N2, int out_dim);
cudaError_t dib_int16_fwd2_head(const void* g_in, int ld_in, int K0, const void* w16_0, const float* b0, const void* w16_1, const float* b1,
                                void* g1, const float* wout, const float* bout, int act, int out_act, float alpha, int loss, const float* y,
                                int M, float inv_batch, float gscale, void* dg2, void* dg1, float* dbpart, void* demb, float* user_pred,
                                float* wpart, int wpart_stride, float* loss_part, float* acc_part, int* nblocks, const float* weights,
                                int bf16, cudaStream_t st);
// head1: the out = 1 kernel (8 rows per pass) instead of the generic one
cudaError_t dib_int16_head(const void* g, int ldg, int K, const float* Wc, const float* bc, int out_dim, int out_act, int hid_act,
                           float alpha, int loss, const float* y, long long n, float inv_batch, float gscale, void* dg, int lddg,
                           float* user_pred, float* wpart, int wpart_stride, float* loss_part, float* acc_part, int nblocks,
                           bool head1, const float* weights, int bf16, cudaStream_t st);

// ---- the set-attention integration network (dib_set_attn.cu; integration_kind 1) ----
// attention core of one block: q, k, v, o (and dout, dq, dk, dv) are [sets * L, heads * dk] with leading dimension ld; lse
// [sets, heads, L] is the row log-sum-exp the forward keeps for the backward.  One CTA per (head, set), L <= 64, dk <= 128.
struct DibAttnArgs {
  const float* q; const float* k; const float* v; int ld;
  float* o; float* lse;
  long long sets; int heads, L, dk;
  int round_out;
  const float* dout; float* dq; float* dk_; float* dv;
  // the key-tiled kernels of sets of different sizes (dib_set_attn_varlen.cu): L is the padded size Lmax, set s has
  // set_sizes[s] real rows; dsum [sets, heads, L] = rowsum(dO o O), written by the query pass of the backward.  Every kernel
  // that reads set sizes takes one outside [1, L] as the nearest bound (dib_set_len)
  const int* set_sizes = nullptr; float* dsum = nullptr;
};
// set-transformer shapes the kernels run: the largest set (fixed-size or key-tiled), heads and key_dim, LayerNorm / pooling E
int dib_attn_max_set_size(bool variable_sizes);
bool dib_attn_heads_ok(int heads, int key_dim);
bool dib_set_width_ok(int E);
size_t dib_attn_smem_bytes(int L, int dk, bool backward);
cudaError_t dib_attn_prepare();   // once per model: the kernels' shared-memory opt-in
cudaError_t dib_launch_attn_fwd(const DibAttnArgs& a, cudaStream_t st);
cudaError_t dib_launch_attn_bwd(const DibAttnArgs& a, cudaStream_t st);
// masked, key-tiled attention of padded sets (shared memory independent of L, dk <= 128); the backward is two launches
cudaError_t dib_attn_varlen_prepare();
cudaError_t dib_launch_attn_varlen_fwd(const DibAttnArgs& a, cudaStream_t st);
cudaError_t dib_launch_attn_varlen_bwd(const DibAttnArgs& a, cudaStream_t st);
// LayerNorm(a + b) over the last axis of [rows, E] (E <= 128, leading dimension ld); mean / rstd [rows] are kept
struct DibLayerNorm {
  const float* a; const float* b; int ld; long long rows; int E;
  const float* gamma; const float* beta; float epsilon;
  float* y; float* mean; float* rstd;
  int round_out;
};
// its backward: dy = sum of dy[0..4) (nullable, [rows, ld]) + dy_pool[row / pool_rows] * pool_scale (nullable);
// d_res = d(a + b); d_branch (nullable) = d_res * act'(b) (b is the output of a Dense with activation branch_act);
// d gamma / d beta partials of CTA s at part + s * split_stride + gamma_off / beta_off, CTA s owning rows_per_split rows
struct DibLayerNormBwd {
  const float* dy[4]; const float* dy_pool; int pool_rows; float pool_scale;
  float* d_res; float* d_branch; int branch_act; float alpha;
  float* part; long long split_stride; long long gamma_off, beta_off; int nsplit; long long rows_per_split;
  // variable set sizes: the pooled source reaches row p of set s as dy_pool[s] / set_sizes[s] for p < set_sizes[s] and not at
  // all for the padding rows (pool_scale is then unused); set_sizes[s] clamped into [1, pool_rows]
  const int* set_sizes = nullptr;
};
cudaError_t dib_launch_ln_fwd(const DibLayerNorm& a, cudaStream_t st);
cudaError_t dib_launch_ln_bwd(const DibLayerNorm& a, const DibLayerNormBwd& b, cudaStream_t st);
// out[s] = mean over the L rows of set s of x [sets * L, ld] (E live columns), out [sets, ldo]
cudaError_t dib_launch_pool_fwd(const float* x, int ld, int E, int L, int64_t sets, float* out, int ldo, int round_out,
                                cudaStream_t st);
// the same over the l_s = sizes[s] real rows of each padded set: out[s] = (sum_{p < l_s} x[s L + p]) / l_s
cudaError_t dib_launch_pool_varlen_fwd(const float* x, int ld, int E, int L, int64_t sets, const int* sizes, float* out, int ldo,
                                       int round_out, cudaStream_t st);
// zero every column of the padding rows p >= sizes[s] of a [rows = sets * L, ld] buffer
cudaError_t dib_launch_zero_pad_rows(float* buf, int ld, int64_t rows, int L, const int* sizes, cudaStream_t st);
// dst[i] = sum of the non-null src[q][i], i < count
struct DibSumRows { const float* src[4]; float* dst; long long count; };
cudaError_t dib_launch_sum_rows(const DibSumRows& a, cudaStream_t st);

cudaError_t dib_launch_mi_sandwich(const float* mu_logvar, int64_t n, int E, const float* eps, uint64_t seed, uint32_t step,
                                   float* row_scratch, float* out2, cudaStream_t st);
// G = features x batches groups of n rows in one launch, float64 accumulation; group g uses the noise stream
// (seed << 8) + g / batches_per_feature at step g % batches_per_feature
cudaError_t dib_launch_mi_sandwich_batched(const float* mu_logvar, int groups, int64_t n, int E, const float* eps, uint64_t seed,
                                           int batches_per_feature, double* row_scratch, double* out, cudaStream_t st);
// per-probe bounds against B batches of data rows [offsets[b], offsets[b+1]) (dib_mi_probes.cu); 1 <= E <= 128, B <= 65535
size_t dib_mi_probes_scratch_bytes(int64_t m, int64_t data_rows, int B, int E);
cudaError_t dib_launch_mi_probes(const float* probes, int64_t m, const float* data, const int64_t* offsets, int B, int E,
                                 const float* eps, uint64_t seed, void* scratch, double* out, cudaStream_t st);
