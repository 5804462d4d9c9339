/* dib_b200_test_hooks.h -- unit-test hooks of libdib_b200.so, apart from the C ABI of dib_b200.h.  Each launches one kernel
 * family through the launcher the library's own steps use, checks its arguments on the host first (failing with a message in
 * dib_last_error() that names the one it rejects) and synchronises the stream. */
#ifndef DIB_B200_TEST_HOOKS_H_
#define DIB_B200_TEST_HOOKS_H_

#include "dib_b200.h"

#ifdef __cplusplus
extern "C" {
#endif

/* unit-test hook: one grouped GEMM launch of the dense-layer kernels, as the library's own steps issue it.
 * A group is `nprob` problem descriptors (host memory; the C mirror of the kernels' descriptor) whose offsets, in floats,
 * are relative to the base pointers: a_off / b_off / c_off to A / B / C, x_off to `bias` (FWD bias), X (DGRAD activation
 * source) or X (WGRAD bias-gradient partials; x_off < 0: none).  Canonical form Out[R x C] = sum_t Aop[R x T] Bop[T x C]:
 *   mode 0 FWD    C = act(A[M x T] B[T x C] + bias)      (T = fan-in,  C = fan-out)
 *   mode 1 DGRAD  C = (A[M x T] B[C x T]^T) * act'(X)    (T = fan-out, C = fan-in; X is the activation output)
 *   mode 2 WGRAD  for each split s: C + s * split_stride = A[rows of s]^T B[rows of s], X + x_off + s * split_stride = the
 *                 column sums of B[rows of s]; split s holds batch rows [s * rows_per_split, min(M, (s + 1) * rows_per_split))
 * maxC / maxR: the largest C / R of the group (grid size).  round_out: round FWD / DGRAD outputs to TF32 (cvt.rna).
 * kernel: DIB_GEMM_KERNEL_SIMT (exact fp32 FMA) or DIB_GEMM_KERNEL_TC (tf32 wgmma); the tensor-core kernel fails with a message
 * on a group it cannot run, it never runs another.  The SIMT kernel reads FWD biases from B's base, so it needs bias == B
 * (or null). */
typedef struct dib_gemm_problem {
  int64_t a_off, b_off, c_off, x_off;
  int32_t lda, ldb, ldc, ldx;
  int32_t T, C, R, act;
} dib_gemm_problem;
enum { DIB_GEMM_KERNEL_SIMT = 0, DIB_GEMM_KERNEL_TC = 1 };
int dib_debug_gemm(int32_t kernel, int32_t mode, const dib_gemm_problem* problems, int32_t nprob, const float* A,
                   const float* B, float* C, float* X, const float* bias, int32_t M, int32_t maxC, int32_t maxR, int32_t nsplit,
                   int32_t rows_per_split, int64_t split_stride, float alpha, int32_t round_out, void* stream);

/* unit-test hook: the streaming InfoNCE sweeps of DIB_LOSS_INFONCE, launched as the library's own steps launch them.
 * kind as dib_scaled_similarity; e1 [n, d] (leading dimension ld1), e2 [n, d] (ld2); the own rows [row0, row0 + rows) of
 * both sides are swept against all n rows of the other side, and rows past n are never read.  phases: 1 = loss sweeps
 * (lse_r[i * lse_stride] = r_i and lse_c[i * lse_stride] = c_i for the own i, diag[i - row0] = s_ii, loss_sum[0] =
 * sum_{own i} (r_i + c_i - 2 s_ii)), 2 = gradient sweeps (read r and c of all n rows from lse_r / lse_c; write d loss / d e1
 * and d loss / d e2 of the own rows at local index, leading dimensions ld_d1 / ld_d2, pad columns zeroed, rounded to TF32
 * when round_out; either may be NULL), 3 = both.  Fails with a message unless 1 <= d <= 512, ld1, ld2 >= d,
 * 0 < temperature < inf, 1 <= n < 2^31, 0 <= row0, 1 <= rows, row0 + rows <= n and lse_stride >= 1. */
int dib_debug_infonce_stream(int32_t kind, float temperature, const float* e1, int32_t ld1, const float* e2, int32_t ld2,
                             int64_t n, int32_t d, int64_t row0, int64_t rows, float* lse_r, float* lse_c, int32_t lse_stride,
                             float* diag, float* loss_sum, float* d_e1, int32_t ld_d1, float* d_e2, int32_t ld_d2,
                             int32_t round_out, int32_t phases, void* stream);

/* unit-test hooks of the set-transformer kernels (DIB_INTEGRATION_SET_TRANSFORMER), with the limits dib_create enforces;
 * tests/test_gpu_set_attention_kernels.py checks them element by element against float64.
 *
 * dib_debug_set_attention: the attention core of one block.  variable_sizes 0: the fixed-size kernels (1 <= L <= 64);
 * 1: the key-tiled masked kernels of padded sets (1 <= L <= DIB_MAX_VARIABLE_SET_SIZE, device int32 set_sizes[sets], each
 * clamped into [1, L]).  q, k, v, dout, o, dq, dk, dv are [sets * L, heads * dk] with leading dimension ld >= heads * dk;
 * lse and dsum are [sets, heads, L].  phases: 1 = forward (o, lse), 2 = backward (dq, dk, dv and, key-tiled, dsum =
 * rowsum(dout o o)) from the o and lse in those buffers, 3 = both.  The key-tiled kernels write zeros to the padding rows of
 * o / dq / dk / dv and to their lse / dsum slots, and never read the padding rows of q / k / v / dout / o.  round_out rounds
 * o / dq / dk / dv to TF32.  Needs 1 <= dk <= 128, heads >= 1, heads * dk a multiple of 4, 0 <= sets <= 65535 (0: nothing
 * is launched). */
int dib_debug_set_attention(int32_t variable_sizes, int32_t phases, const float* q, const float* k, const float* v,
                            const float* dout, int32_t ld, int64_t sets, int32_t heads, int32_t L, int32_t dk,
                            const int32_t* set_sizes, float* o, float* lse, float* dq, float* dk_grad, float* dv, float* dsum,
                            int32_t round_out, void* stream);

/* dib_debug_layer_norm: y = LayerNorm(a + b) over the E live columns of [rows, ld] rows (biased variance; mean / rstd [rows]
 * kept), and / or its backward from caller-supplied mean / rstd.  phases: 1 = forward, 2 = backward, 3 = both.  The backward's
 * dy = dy0 + dy1 + dy2 + dy3 (each nullable, [rows, ld]) + the pooled source: dy_pool [rows / pool_rows, ld] times
 * fl(1 / pool_rows) on every row, or, with set_sizes, times 1 / l_s on the l_s real rows of each set of pool_rows rows and
 * nothing on its padding rows.  d_res = d(a + b); d_branch (nullable) = d_res * act'(b) for the activation branch_act
 * (derivative from the output b, leaky slope alpha).  Split s covers rows [s * rows_per_split, (s + 1) * rows_per_split)
 * and writes its d gamma / d beta partials (zero for a split past the rows) to part + s * split_stride + gamma_off / beta_off.
 * y, d_res and d_branch get zeros in their columns E <= e < min(ld, 128).  Needs 1 <= E <= 128 a multiple of 4, ld >= E,
 * 0 <= epsilon < inf,
 * and for the backward nsplit * rows_per_split >= rows with both partial ranges inside [0, split_stride). */
int dib_debug_layer_norm(int32_t phases, const float* a, const float* b, int32_t ld, int64_t rows, int32_t E, const float* gamma,
                         const float* beta, float epsilon, float* y, float* mean, float* rstd, const float* dy0,
                         const float* dy1, const float* dy2, const float* dy3, const float* dy_pool, int32_t pool_rows,
                         const int32_t* set_sizes, float* d_res, float* d_branch, int32_t branch_act, float alpha, float* part,
                         int64_t split_stride, int64_t gamma_off, int64_t beta_off, int32_t nsplit, int64_t rows_per_split,
                         int32_t round_out, void* stream);

/* dib_debug_set_pool: zero_pad 0 = out [sets, ldo] = the mean over the L rows of each set of x [sets * L, ld] (E live
 * columns; out's columns E <= e < ldo zeroed), or with set_sizes over its l_s real rows; zero_pad 1 = zero every column of
 * the padding rows p >= l_s of x (out unused).  l_s = set_sizes[s] clamped into [1, L].  Needs 1 <= L <= 64 (fixed) or
 * DIB_MAX_VARIABLE_SET_SIZE (with set_sizes), 0 <= sets <= 65535, and for the mean 1 <= E <= 128 a multiple of 4, ld >= E,
 * ldo >= E. */
int dib_debug_set_pool(int32_t zero_pad, float* x, int32_t ld, int32_t E, int32_t L, int64_t sets, const int32_t* set_sizes,
                       float* out, int32_t ldo, int32_t round_out, void* stream);

/* unit-test hooks of the elementwise kernels of every training step (csrc/dib_elementwise.cu), with the limits dib_create
 * enforces; tests/test_gpu_elementwise_kernels.py checks them element by element against float64.
 *
 * dib_debug_reparam: phases 1 = forward: emb[row, f E + e] = u = mu + exp(lv / 2) z (TF32-rounded when round_out; columns
 * F E <= c < ldemb zeroed), user_emb [n, F E] (nullable) = u unrounded, kl_part[f * nblk_stride + b] = the KL of feature f summed
 * over the 256 rows of block b; 2 = backward: d_out (enc_out's layout) = (du + beta inv_batch mu | du z sigma / 2 + beta inv_batch
 * expm1(lv) / 2 | zeros up to ldo) from d_emb [n, ldemb] and beta_dev[0]; 3 = both.  enc_out: feature f's row r is
 * (mu[E] | lv[E] | pad) at f * feat_stride + r * ldo.  z = eps[(r F + f) E + e] when eps is given, else the Philox normal of
 * (seed, step + *step_dev, sample_offset + r, f).  With set_sizes (device int32, n / set_len sets, each clamped into
 * [1, set_len]) a padding row gets u = 0, no KL and a zero gradient.  Needs 1 <= F <= 65535, E >= 1, ldo >= 2E,
 * feat_stride >= n ldo, ldemb >= F E, 0 <= n < 2^31, nblk_stride >= ceil(n / 256) and 1 <= set_len <= DIB_MAX_VARIABLE_SET_SIZE
 * dividing n. */
int dib_debug_reparam(int32_t phases, const float* enc_out, int64_t feat_stride, int32_t ldo, int32_t F, int32_t E, int64_t n,
                      const float* eps, uint64_t seed, uint32_t step, const uint32_t* step_dev, uint64_t sample_offset,
                      const int32_t* set_sizes, int32_t set_len, float* emb, int32_t ldemb, float* user_emb, float* kl_part,
                      int32_t nblk_stride, const float* d_emb, const float* beta_dev, float inv_batch, float* d_out,
                      int32_t round_out, void* stream);

/* dib_debug_loss: the compiled loss of n rows of pred [n, ldp] (out_dim live columns) against y (sparse CE: [n] labels, the
 * external loss: d task loss / d pred [n, out_dim], else [n, out_dim]; NULL: no loss) with the output activation out_act
 * (derivative from the output): d_pred [n, ldp] (nullable; columns out_dim <= c < ldp zeroed), user_pred [n, out_dim]
 * (nullable), and per 256-row block b loss_part[b] / acc_part[b] = the block's sums of the rows' loss and accuracy.  weights
 * (nullable, not with DIB_LOSS_EXTERNAL): the rows' sample weights.  Needs loss != DIB_LOSS_INFONCE, a known out_act,
 * out_dim >= 1, ldp >= out_dim and 0 <= n < 2^31. */
int dib_debug_loss(int32_t loss, int32_t out_act, float alpha, const float* pred, int32_t ldp, const float* y, int32_t out_dim,
                   int64_t n, float inv_batch, const float* weights, float* d_pred, float* user_pred, float* loss_part,
                   float* acc_part, int32_t round_out, void* stream);

/* dib_debug_reduce: kind 0 = the batch-split partial sum: dst[i] = sum_{k < nrows} src[k row_stride + i], i < count;
 * kind 1 = the nseg segments (host array) of one fixed-order reduction list, as the training step hands it over: segment s
 * writes dst[i] = scale sum_{k < nrows} src[k row_stride + i] for i < count, and a segment with count <= 0 is skipped; the
 * list runs as ceil(live segments / 8) launches; kind 2 = the step statistics: dst[f] = sum_{b < count} src[f row_stride + b]
 * for f < nrows = F, dst[F] / dst[F + 1] = the sums of loss_part / acc_part [nblk_loss] (0 unless has_y), dst[F + 2] = n.
 * Needs count >= 0, nrows >= 0 (kind 2: >= 1), row_stride >= count and count < 2^31 in every reduction. */
typedef struct dib_reduce_seg {
  const float* src;
  int64_t row_stride;
  int32_t nrows;
  int64_t count;
  float scale;
  float* dst;
} dib_reduce_seg;
int dib_debug_reduce(int32_t kind, const float* src, int64_t row_stride, int32_t nrows, int64_t count, float* dst,
                     const dib_reduce_seg* segs, int32_t nseg, const float* loss_part, const float* acc_part, int32_t nblk_loss,
                     int64_t n, int32_t has_y, void* stream);

/* dib_debug_pe: the positional encoding of the step into pe [n, ldpe]: for every column col in [col_begin, col_end) of the
 * device tables col_src / col_freq (/ col_feat), pe[r, col - pe_col_shift] = 0 when col_src[col] < 0, else with
 * x~ = x[r', col_src[col] - x_col_shift] (r' = r, or with row_index the row row_index[col_feat[col] n + r] clamped into
 * [0, n_src)) x~ itself when col_freq[col] = 0 and sinf(col_freq[col] x~) otherwise; TF32-rounded when round_out.  The hook reads
 * the tables and needs every column to land inside [0, ldpe) and every source inside [0, ldx), n >= 0 and, with row_index,
 * col_feat and n_src >= 1 (row_index holds (max col_feat + 1) n entries). */
int dib_debug_pe(const float* x, int32_t ldx, int32_t x_col_shift, const int32_t* col_src, const int32_t* col_freq,
                 int32_t col_begin, int32_t col_end, float* pe, int32_t ldpe, int32_t pe_col_shift, int64_t n,
                 const int32_t* row_index, const int32_t* col_feat, int64_t n_src, int32_t round_out, void* stream);

/* dib_debug_dropout: Keras Dropout of the encoder activations: dst = src keep / (1 - rate) (backward: dst *= the same mask,
 * in place; src unused) over the width live columns of row r of feature f at f feat_stride + r ld, for every feature
 * (feature = -1) or one; the keep mask of (seed, step + *step_dev, sample_offset + r, f, layer) is oracle/philox.dropout_keep.
 * Needs 0 <= rate < 1, width >= 1, ld >= width, feat_stride >= n ld, 1 <= F <= 65535, -1 <= feature < F, 0 <= layer < 128. */
int dib_debug_dropout(const float* src, float* dst, int64_t feat_stride, int32_t ld, int32_t width, int32_t F, int64_t n,
                      float rate, uint64_t seed, uint32_t step, const uint32_t* step_dev, uint64_t sample_offset, int32_t layer,
                      int32_t feature, int32_t backward, int32_t round_out, void* stream);

/* unit-test hooks of the 16-bit integration network kernels (csrc/dib_int16.cu: 'fp16' / 'bf16' precision).  bf16: 0 = fp16
 * operands, 1 = bf16.  16-bit buffers hold raw fp16 / bf16 bit patterns.  Every 16-bit base must be 16-byte aligned and every 16-bit leading dimension a multiple of 8 and no smaller
 * than the width it holds (the TMA descriptors and the vector accesses need both); fp32 bias rows must be 8-byte aligned.
 * Widths are what dib_create allows: the embedding width a multiple of 64, hidden widths multiples of 128.
 * tests/test_gpu_int16_kernels.py checks them element by element against a float64 reference.
 *
 * dib_debug_int16_gemm: mode 0 FWD   out [M, N] (ldc) = r(act(a [M, K] (lda) w16 [K, N] + bias [N]))
 *                       mode 1 DGRAD out [M, K] (ldc) = r((a [M, N] (lda) w16 [K, N]^T) act'(x [M, K] (ldx))), x nullable (no
 *                              act'); colsum (nullable) [ceil(M / 128)][K] = the column sums of the unrounded result per
 *                              128-row tile
 *                       mode 2 WGRAD for each of the `count` (1 or 2) layers and split s < nsplit: layers[q].dW_part +
 *                              s * split_stride = out_scale g_in[rows of s]^T dz[rows of s] [K x N], g_in [M, K] and dz [M, N]
 *                              dense; split s holds batch rows [s rows_per_split, min(M, (s + 1) rows_per_split)), a split
 *                              past M writes zeros.  Needs rows_per_split > 0 a multiple of 64 (a k-block of 64 rows must
 *                              not reach into the next split), nsplit rows_per_split >= M, and K N <= split_stride.
 * r() is cvt.rn.satfinite to the 16-bit format.  Needs K % 64 == 0, N % 128 == 0 and M >= 1. */
typedef struct dib_int16_wgrad_layer {
  const void* g_in;
  int32_t K;
  const void* dz;
  int32_t N;
  float* dW_part;
  int32_t nsplit;
  int32_t rows_per_split;
} dib_int16_wgrad_layer;
int dib_debug_int16_gemm(int32_t mode, int32_t bf16, int32_t M, int32_t K, int32_t N, const void* a, int32_t lda,
                         const void* w16, const float* bias, const void* x, int32_t ldx, void* out, int32_t ldc, int32_t act,
                         float alpha, float* colsum, const dib_int16_wgrad_layer* layers, int32_t count, int64_t split_stride,
                         float out_scale, void* stream);

/* dib_debug_int16_head: the output head over n rows of the last hidden activation g [n, K] (ldg), K = 256: z = out_act(g Wc +
 * bc) (Wc [K, out_dim], bc [out_dim] fp32), the compiled loss against y (nullable), and in training (dg != NULL) dg [n, K]
 * (lddg) = r(dz S Wc^T act'(g)) plus per-block partials wpart[b * wpart_stride + ...] = [dWc (K out) | dbc (out) | column sums
 * of dg (K)]; loss_part[b] / acc_part[b] for each of the nblocks blocks; user_pred [n, out_dim] (nullable) = z.  head1: the
 * out = 1 kernel.  weights (nullable): the rows' sample weights.  Needs 1 <= out_dim <= 16, head1 => out_dim == 1, n >= 1,
 * nblocks >= 1 and, in training, wpart_stride >= K out + out + K. */
int dib_debug_int16_head(int32_t head1, int32_t bf16, const void* g, int32_t ldg, int32_t K, const float* Wc, const float* bc,
                         int32_t out_dim, int32_t out_act, int32_t hid_act, float alpha, int32_t loss, const float* y, int64_t n,
                         float inv_batch, float gscale, void* dg, int32_t lddg, float* user_pred, float* wpart,
                         int32_t wpart_stride, float* loss_part, float* acc_part, int32_t nblocks, const float* weights,
                         void* stream);

/* dib_debug_int16_fwd2: the fused tail of single-output models: g1 [M, 256] = r(act(g_in [M, K0] (ld_in) W0 + b0)),
 * g2 = r(act(g1 W1 + b1)) on chip, the logit and compiled loss; training (dg2 != NULL): dg2 [M, 256] and the per-CTA
 * partials wpart[b * wpart_stride + ...] = [dW out (256) | db out (1) | column sums of dg2 (256)]; with dg1 (needs dg2 and
 * dbpart) the dgrad of the second layer dg1 [M, 256] with its column sums per 128-row tile in dbpart [ceil(M / 128)][256];
 * with demb (needs dg1) demb [M, K0] = r(dg1 W0^T).  *nblocks = the CTAs launched (rows of wpart / loss_part / acc_part
 * written).  Needs K0 % 64 == 0 (K0 >= 64), n >= 1 and, in training, wpart_stride >= 513. */
int dib_debug_int16_fwd2(int32_t bf16, const void* g_in, int32_t ld_in, int32_t K0, const void* w16_0, const float* b0,
                         const void* w16_1, const float* b1, void* g1, const float* wout, const float* bout, int32_t act,
                         int32_t out_act, float alpha, int32_t loss, const float* y, int32_t M, float inv_batch, float gscale,
                         void* dg2, void* dg1, float* dbpart, void* demb, float* user_pred, float* wpart, int32_t wpart_stride,
                         float* loss_part, float* acc_part, const float* weights, int32_t* nblocks, void* stream);

/* dib_debug_enc_fused: the fused per-feature encoder kernels of the 'fp16' / 'bf16' precision (csrc/dib_enc_fused.cu), launched
 * through the launchers the step uses; phases is a mask: 1 = pack the fp32 params into the 16-bit image `packed` (bias
 * carriers, b2's logvar half + logvar_offset), and clear kl_part [F][kl_stride] when the pack grid covers it; 2 = forward:
 * per row r < n and feature f, emb[r, 32 f + e] = TF32(u), user_emb[r, 32 f + e] = u, emb16 = r(u) (each nullable),
 * u = mu + exp(lv / 2) eps, and kl_part[f kl_stride + slot] = the KL sum of the slot's rows; 4 = backward from d_emb [n, ldd]
 * (fp32, times gscale) or d_emb16 [n, ldd16] (16-bit, already times gscale) -- exactly one -- into the weight-gradient
 * partials part[slot split_stride + the parameter offsets].  The feature f has fdim[f] (1..3) x columns from x_off[f] of x
 * [n, ldx], nfreq - 1 sinusoid blocks, and its parameters at the host tables w0_off .. b2_off in the model's layout (W0
 * [fdim nfreq, 128], b0 [128], W1 [128, 128], b1 [128], W2 [128, 64], b2 [64]).  eps [n, F, 32] or, when null, the Philox
 * noise of (seed, step + *step_dev, sample_offset + r).  grid 0 is the library's choice per phase (forward min(F tiles,
 * 2 SMs), backward min(F tiles, SMs)); otherwise 1 <= grid <= F ceil(n / 128), the same for both phases.  With grid >= F
 * CTA c serves feature c % F and its tiles c / F, c / F + nslots, ...; with grid < F it walks features c, c + grid, ....
 * Slot rows of a feature served by fewer CTAs are not written (the step clears them).  Needs fdim nfreq + 1 <= 16, x columns
 * and parameter blocks in range (and, in the backward, inside split_stride), even leading dimensions and 8-byte bases for the
 * float2 accesses, a 16-byte d_emb16 with ldd16 a multiple of 8 and >= 32 F, kl_stride >= ceil(grid / F), gscale a power of
 * two.
 * tests/test_gpu_enc_fused_kernels.py checks the kernels element by element against a float64 reference. */
int dib_debug_enc_fused(int32_t phases, int32_t F, const int32_t* fdim, const int32_t* x_off, int32_t nfreq, int32_t act,
                        float alpha, int32_t bf16, float logvar_offset, const float* params, int64_t param_count,
                        const int64_t* w0_off, const int64_t* b0_off, const int64_t* w1_off, const int64_t* b1_off,
                        const int64_t* w2_off, const int64_t* b2_off, int32_t grid, int64_t n, const float* x, int32_t ldx,
                        const float* eps, uint64_t seed, uint32_t step, const uint32_t* step_dev, uint64_t sample_offset,
                        float* emb, int32_t ldemb, float* user_emb, void* emb16, int32_t ldemb16, float* kl_part,
                        int32_t kl_stride, const float* d_emb, int32_t ldd, const void* d_emb16, int32_t ldd16,
                        const float* beta_dev, float inv_batch, float gscale, float* part, int64_t split_stride, void* packed,
                        void* stream);

#ifdef __cplusplus
}
#endif
#endif /* DIB_B200_TEST_HOOKS_H_ */
