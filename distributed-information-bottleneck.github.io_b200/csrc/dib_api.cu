// dib_api.cu -- the C ABI declared in include/dib_b200.h: model description, workspace plan, and the
// orchestration of one forward / train step as a fixed sequence of asynchronous launches on the caller's stream.
#include <atomic>
#include <cmath>
#include <cstddef>
#include <cstdio>
#include <cstring>
#include <new>
#include <string>
#include <vector>

#include "dib_common.cuh"
#include "dib_kernels.h"

namespace {

thread_local std::string g_last_error;
std::atomic<unsigned long long> g_launches{0};

int fail(const std::string& msg) {
  g_last_error = msg;
  return 1;
}

#define DIB_CUDA_OK(expr)                                                                        \
  do {                                                                                           \
    cudaError_t _e = (expr);                                                                     \
    if (_e != cudaSuccess)                                                                       \
      return fail(std::string(#expr) + ": " + cudaGetErrorString(_e));                           \
  } while (0)

struct Buf {
  long long off = 0;          // float offset inside the workspace
  int ld = 0;                 // leading dimension (multiple of 4)
  long long feat_stride = 0;  // distance between consecutive features (0 for single matrices)
};

// a stack of Dense layers 0..L on the per-layer grouped GEMMs (dib_gemm_simt.cu in fp32, dib_gemm_tc.cu otherwise): every
// layer is one launch per GEMM mode over G groups -- the F feature encoders, Q / K / V, else one.  build_stack emits its
// problems, stack_forward / stack_backward run them.
struct Stack {
  int G = 1;
  std::vector<int> fwd, dgrad, wgrad;   // [j]: first of layer j's G problems in d_probs (dgrad[0] = -1 without dgrad0)
  std::vector<int> fan_in, fan_out;     // [j]: largest fan-in over the groups (DGRAD maxC, WGRAD maxR), fan-out
  bool dgrad0 = false;                  // layer 0 has a DGRAD: the gradient of the stack's input is wanted
  float drop = 0.f;                     // Keras Dropout after every hidden layer (the feature encoders only)
  const char* label = nullptr;          // profile ranges <label>_fwd_l<j> ...; none: the stack runs inside its caller's range
};

constexpr int kMaxSplits = 32;
constexpr int kRowsPerBlock = 256;

}  // namespace

struct dib_model {
  int F = 0, L = 0, Li = 0, E = 0, D = 0, out = 0;
  int act = 0, out_act = 0, loss = 0, precision = 0, use_pe = 0, nfreq = 1;
  float alpha = 0.2f;
  long long maxB = 0;
  std::vector<int> fdims, enc_arch, int_arch;
  std::vector<int> x_off, pe_off, w_in;  // per feature: x column, pe column, first-layer fan-in
  int ldpe = 0;
  // parameters
  long long P = 0, Pp = 0;
  std::vector<long long> var_off;
  std::vector<int> var_rows, var_cols;
  std::vector<std::vector<long long>> encW, encB;  // [f][j]
  std::vector<long long> intW, intB;               // [j]
  // workspace plan
  long long ws_floats = 0;
  Buf pe, enc_out, emb, pred, d_pred, d_emb, d_out;
  std::vector<Buf> enc_act, d_enc;  // index 1..L  (output of layer j-1)
  std::vector<Buf> enc_drop;        // index 1..L  (dropout_rate > 0: what layer j reads -- enc_act[j] after Keras Dropout)
  float drop = 0.f;
  std::vector<Buf> int_act, d_int;  // index 1..Li
  long long part_off = 0, kl_part_off = 0, loss_part_off = 0, acc_part_off = 0, wshadow_off = 0;
  int nblk_max = 0;
  // device tables
  DibGemmProblem* d_probs = nullptr;
  std::vector<DibGemmProblem> h_probs;
  int* d_col_src = nullptr;
  int* d_col_freq = nullptr;
  int* d_col_feat = nullptr;   // feature owning each first-layer operand column (row gather of dib_compression_matrices)
  Stack enc_stack, int_stack;  // the feature encoders (not the SimpleEncoder), the integration network / set-transformer head
  // fused per-feature encoder kernels (tensor-core mode; dib_enc_fused.cu)
  bool fused_ok = false;
  DibEncFusedDesc fdesc;
  void* d_fused_tables = nullptr;
  long long pack_off = 0;       // packed 16-bit encoder weights inside the workspace (float offset)
  int kl_stride = 0, num_sms = 132, part_rows = kMaxSplits;
  // 16-bit integration network path (dib_int16.cu); offsets are FLOAT offsets into the workspace
  bool int16_ok = false;
  long long emb16_off = 0, demb16_off = 0, headpart_off = 0, dbpart_off = 0;
  int head_stride = 0, dbpart_stride = 0;
  long long dbpart_layer = 0;       // floats per layer of the dgrad column-sum partials
  std::vector<long long> g16_off, dg16_off, w16_off;   // [1..Li], [1..Li], [0..Li-1]
  int head_blocks = 0, lossacc_cap = 0;
  int head_used = 0;                // rows of the head partials the last forward wrote (fused tail kernel: its CTA count)
  // the kernels this handle runs (set_route): every forward / backward / dib_model_info reads the choice from here
  struct Route {
    bool enc_fused = false;         // fused per-feature encoder kernels (else PE + grouped GEMMs + reparam kernels)
    bool int16 = false;             // 16-bit integration network (else per-layer TF32 GEMMs + dib_launch_loss)
    bool tail_fused = false;        // int16: last two hidden layers + head + loss as one kernel (dib_int16_fwd2_head)
    bool tail_bwd = false;          // tail_fused, training: the same kernel also runs the dgrad of its second layer (and of
                                    // its first when the embedding lies below), which the backward then does not launch
    bool head1 = false;             // int16, no fused tail: the out = 1 head kernel instead of the generic one
  } route;
  // DIB_LOSS_INFONCE (train.py:180-289): the output encoder y -> [PE] -> Dense(y_arch[j], act)... -> Dense(out), its variables
  // after the model's in the flat buffer, and the streaming InfoNCE loss (dib_infonce_stream.cu)
  long long Px = 0;                 // end of the model's own parameters (== P without an output encoder)
  int ydim = 0, Ly = 0, sim_kind = 0, ldype = 0;
  float temperature = 1.f;
  std::vector<int> y_arch;
  std::vector<long long> yW, yB;    // [j]
  Buf ype, y_out, d_y_out;          // PE(y), e2 = output_encoder(y), d loss / d e2
  std::vector<Buf> y_act, d_yact;   // index 1..Ly
  long long nce_off = 0;            // 3 * max_batch floats of InfoNCE scratch
  long long nce_stats_off = 0;      // F + 3 floats: the stats dib_infonce_shard_lse wrote, for the backward's IB weight
  int nce_nblk_kl = 0;              // KL partials per feature dib_infonce_shard_forward left for dib_infonce_shard_lse
  Stack y_stack;
  int* d_ycol_src = nullptr;
  int* d_ycol_freq = nullptr;
  // DIB_INTEGRATION_SET_TRANSFORMER (nb-particle cell 8, dib_set_attn.cu): the encoder and the attention blocks run on
  // n * Ls particle rows (maxB counts rows, maxSets sets), the head on the n set means
  bool st = false;
  int Ls = 1, nblk = 0, heads = 0, dkey = 0, hdk = 0, ff_act = 0;
  // variable set sizes (dib_config.variable_set_sizes): Ls is the padded size Lmax and the caller binds the int32 sizes of the
  // n sets of the following calls (dib_set_set_sizes_device); the attention runs on the key-tiled kernels of
  // dib_set_attn_varlen.cu, which keep rowsum(dO o O) at dsum between their two backward passes
  bool varlen = false;
  const int32_t* set_sizes_dev = nullptr;
  long long dsum = 0;
  // per-row sample weights of the following dib_forward / dib_train_step calls (dib_set_sample_weights_device), or null
  const float* sample_weights_dev = nullptr;
  // compiled metrics (dib_set_metrics): their table and, behind the planned workspace (plan_floats), the prediction
  // [rows, out] the loss kernels write for them and the metric kernel's CTA partials; the last CTA's counter
  DibMetricTable metrics;
  long long plan_floats = 0, metric_z_off = 0, metric_part_off = 0;
  unsigned int* d_metric_counter = nullptr;
  float ln_eps = 1e-3f;
  long long maxSets = 0;
  std::vector<int> ff_arch;
  struct StBlock {
    long long Wq, bq, Wk, bk, Wv, bv, Wo, bo, g1, be1, g2, be2;
    std::vector<long long> ffW, ffB;                  // [j]
    Buf q, k, v, o, a, hh, xout;                      // Q, K, V, attention output (heads concatenated), its projection, LN1, LN2
    std::vector<Buf> ff;                              // index 1..nff: output of FF layer j-1
    long long lse = 0, mean1 = 0, rstd1 = 0, mean2 = 0, rstd2 = 0;
    Stack qkv_stack, o_stack, ff_stack;               // Q / K / V (G = 3), the output projection, the FF stack
  };
  std::vector<StBlock> blk;
  Buf dq, dk, dv, d_o, dz1, dz2, dh_ff, dxq, dxk, dxv, pooled, d_pooled;   // backward scratch shared by the blocks
  std::vector<Buf> d_ff;                             // index 1..nff
  // custom-step variants (SURVEY 8f3)
  float lv_off = 0.f, kl_exp = 1.f, kl_scale = 1.f;
  const uint32_t* step_dev = nullptr;  // optional device-resident addend of the Philox step word (dib_set_noise_step_device)
  bool simple = false;                 // nb-bool SimpleEncoder: two (1,1) constants per feature
  int* d_xoff = nullptr;               // device copy of x_off (simple-encoder kernels)
  long long beta_eff_off = 0;          // one float in the workspace: d(beta*scale*KL^p)/dKL
  // optional per-launch-group timing with CUDA events on the caller's stream (dib_profile_*)
  bool profiling = false;
  struct ProfRec { std::string label; cudaEvent_t a, b; };
  std::vector<ProfRec> prof;
};

namespace {

// precision modes: FP32 = CUDA-core FMA; TF32 = tf32 wgmma grouped GEMMs on fp32 storage; FP16 / BF16 = the fused
// 16-bit-operand kernels (dib_enc_fused.cu, dib_int16.cu) where the shapes allow, tf32 GEMMs elsewhere
bool is_tc(const dib_model* h) { return h->precision != DIB_PREC_FP32; }
bool want16(const dib_model* h) { return h->precision == DIB_PREC_FP16 || h->precision == DIB_PREC_BF16; }

int enc_fan_in(const dib_model* h, int f, int j) { return j == 0 ? h->w_in[f] : h->enc_arch[j - 1]; }
int enc_fan_out(const dib_model* h, int j) { return j < h->L ? h->enc_arch[j] : 2 * h->E; }
int int_fan_in(const dib_model* h, int j) { return j == 0 ? h->F * h->E : h->int_arch[j - 1]; }
int int_fan_out(const dib_model* h, int j) { return j < h->Li ? h->int_arch[j] : h->out; }
bool infonce(const dib_model* h) { return h->loss == DIB_LOSS_INFONCE; }
int y_fan_in(const dib_model* h, int j) { return j == 0 ? h->ydim * h->nfreq : h->y_arch[j - 1]; }
int y_fan_out(const dib_model* h, int j) { return j < h->Ly ? h->y_arch[j] : h->out; }
int ff_fan_in(const dib_model* h, int j) { return j == 0 ? h->E : h->ff_arch[j - 1]; }
int nff(const dib_model* h) { return (int)h->ff_arch.size(); }

// the one place the kernel path is chosen.  fused_ok / int16_ok are what dib_create found the shapes to support; the bits of
// `unfused` (dib_debug_force_unfused) turn paths off: 1 = fused encoders, 2 = 16-bit integration network (it reads the fp16
// embedding only the fused encoders write), 4 = fused integration tail, 8 = out = 1 head kernel, 16 = the dgrad stages of
// the fused tail (separate dgrad launches instead).
void set_route(dib_model* h, int unfused) {
  dib_model::Route& r = h->route;
  r.enc_fused = h->fused_ok && !(unfused & 1);
  r.int16 = r.enc_fused && h->int16_ok && !(unfused & 2);
  r.tail_fused = r.int16 && !(unfused & 4) && h->Li >= 2 &&
                 dib_int16_fwd2_ok(int_fan_in(h, h->Li - 2), int_fan_out(h, h->Li - 2), int_fan_out(h, h->Li - 1), h->out);
  r.tail_bwd = r.tail_fused && !(unfused & 16);
  r.head1 = r.int16 && !r.tail_fused && h->out == 1 && !(unfused & 8);
}

// power-of-two loss scale of the 16-bit gradient operands (see dib_enc_fused.cu)
float loss_scale(float inv_batch) { return exp2f(ceilf(log2f(1.f / inv_batch))); }

// deterministic split of the batch for the weight gradients
struct Split { long long rps; int nsplit; };
Split batch_split(long long n) {
  long long rps = DIB_CEIL_DIV(n, (long long)kMaxSplits);
  if (rps < 256) rps = 256;
  rps = DIB_ROUND_UP(rps, 64);      // whole k-blocks of every WGRAD kernel (32 rows for the TF32 ones, 64 for the 16-bit ones)
  return {rps, (int)DIB_CEIL_DIV(n, rps)};
}

long long take(long long& cursor, long long floats) {
  const long long off = cursor;
  cursor += DIB_ROUND_UP(floats, 64);   // 256-byte granularity
  return off;
}

Buf make_buf(long long& cursor, long long rows, int width, int nfeat) {
  Buf b;
  b.ld = DIB_ROUND_UP(width, 4);
  b.feat_stride = DIB_ROUND_UP(rows * b.ld, 64);
  b.off = take(cursor, b.feat_stride * nfeat);
  return b;
}

void plan(dib_model* h) {
  long long c = 0;
  const long long B = h->maxB;
  h->pe = make_buf(c, B, h->ldpe, 1);
  h->pe.ld = h->ldpe;
  h->enc_act.assign(h->L + 1, Buf());
  h->d_enc.assign(h->L + 1, Buf());
  for (int j = 1; j <= h->L; ++j) h->enc_act[j] = make_buf(c, B, h->enc_arch[j - 1], h->F);
  h->enc_drop.assign(h->L + 1, Buf());
  for (int j = 1; j <= h->L && h->drop > 0.f; ++j) h->enc_drop[j] = make_buf(c, B, h->enc_arch[j - 1], h->F);
  h->enc_out = make_buf(c, B, 2 * h->E, h->F);
  h->emb = make_buf(c, B, h->F * h->E, 1);
  h->int_act.assign(h->Li + 1, Buf());
  h->d_int.assign(h->Li + 1, Buf());
  const long long Bi = h->st ? h->maxSets : B;    // rows of the integration network (the set transformer's head: sets)
  for (int j = 1; j <= h->Li; ++j) h->int_act[j] = make_buf(c, Bi, h->int_arch[j - 1], 1);
  h->pred = make_buf(c, Bi, h->out, 1);
  // backward
  h->d_pred = make_buf(c, Bi, h->out, 1);
  for (int j = 1; j <= h->Li; ++j) h->d_int[j] = make_buf(c, Bi, h->int_arch[j - 1], 1);
  h->d_emb = make_buf(c, B, h->F * h->E, 1);
  h->d_out = make_buf(c, B, 2 * h->E, h->F);
  for (int j = 1; j <= h->L; ++j) h->d_enc[j] = make_buf(c, B, h->enc_arch[j - 1], h->F);
  h->nblk_max = (int)DIB_CEIL_DIV(B, (long long)kRowsPerBlock);
  h->part_rows = DIB_CEIL_DIV(h->num_sms, h->F) > kMaxSplits ? DIB_CEIL_DIV(h->num_sms, h->F) : kMaxSplits;
  h->part_off = take(c, (long long)h->part_rows * h->Pp);
  h->kl_stride = h->nblk_max > 2 * h->num_sms + 8 ? h->nblk_max : 2 * h->num_sms + 8;   // >= fused-kernel CTA slots per feature
  h->kl_part_off = take(c, (long long)h->F * h->kl_stride);
  h->head_blocks = dib_int16_head_blocks(h->num_sms);
  h->lossacc_cap = h->nblk_max > h->head_blocks ? h->nblk_max : h->head_blocks;
  h->loss_part_off = take(c, h->lossacc_cap);
  h->acc_part_off = take(c, h->lossacc_cap);
  {
    const long long FE = (long long)h->F * h->E;
    h->emb16_off = take(c, (B * FE + 1) / 2);
    h->demb16_off = take(c, (B * FE + 1) / 2);
    h->g16_off.assign(h->Li + 1, 0); h->dg16_off.assign(h->Li + 1, 0); h->w16_off.assign(h->Li + 1, 0);
    for (int j = 1; j <= h->Li; ++j) {
      h->g16_off[j] = take(c, (B * h->int_arch[j - 1] + 1) / 2);
      h->dg16_off[j] = take(c, (B * h->int_arch[j - 1] + 1) / 2);
    }
    for (int j = 0; j < h->Li; ++j) h->w16_off[j] = take(c, ((long long)int_fan_in(h, j) * int_fan_out(h, j) + 1) / 2);
    const int Kh = h->Li ? h->int_arch[h->Li - 1] : 1;
    h->head_stride = Kh * h->out + h->out + Kh;          // [dWc | dbc | column sums of dg (bias grad of the last hidden layer)]
    h->headpart_off = take(c, (long long)h->head_blocks * h->head_stride);
    int wmax = 1;
    for (int j = 0; j < h->Li; ++j) if (h->int_arch[j] > wmax) wmax = h->int_arch[j];
    h->dbpart_stride = wmax;                             // dgrad-epilogue column sums: [row tile][width]
    h->dbpart_layer = DIB_ROUND_UP((long long)DIB_CEIL_DIV(B, 128ll) * wmax, 64);
    h->dbpart_off = take(c, h->dbpart_layer * (h->Li > 0 ? h->Li : 1));    // one region per layer: all reduced in one launch
  }
  h->beta_eff_off = take(c, 64);
  h->wshadow_off = take(c, h->Pp);      // TF32-rounded copy of the parameters (tensor-core mode B operands)
  h->pack_off = take(c, (long long)(dib_enc_fused_pack_bytes(h->F) + 3) / 4);
  if (infonce(h)) {                     // the output encoder's activations and gradients, the InfoNCE scratch: all O(max_batch)
    h->ype = make_buf(c, B, h->ldype, 1);
    h->y_act.assign(h->Ly + 1, Buf());
    h->d_yact.assign(h->Ly + 1, Buf());
    for (int j = 1; j <= h->Ly; ++j) h->y_act[j] = make_buf(c, B, h->y_arch[j - 1], 1);
    h->y_out = make_buf(c, B, h->out, 1);
    h->d_y_out = make_buf(c, B, h->out, 1);
    for (int j = 1; j <= h->Ly; ++j) h->d_yact[j] = make_buf(c, B, h->y_arch[j - 1], 1);
    h->nce_off = take(c, 3 * B);
    h->nce_stats_off = take(c, h->F + 3);
  }
  if (h->st) {                          // per block what its backward reads; one set of backward scratch for all blocks
    const int E = h->E, nf = nff(h);
    for (auto& b : h->blk) {
      b.q = make_buf(c, B, h->hdk, 1); b.k = make_buf(c, B, h->hdk, 1); b.v = make_buf(c, B, h->hdk, 1);
      b.o = make_buf(c, B, h->hdk, 1);
      b.lse = take(c, h->maxSets * h->heads * h->Ls);
      b.a = make_buf(c, B, E, 1);
      b.mean1 = take(c, B); b.rstd1 = take(c, B);
      b.hh = make_buf(c, B, E, 1);
      b.ff.assign(nf + 1, Buf());
      for (int j = 1; j <= nf; ++j) b.ff[j] = make_buf(c, B, h->ff_arch[j - 1], 1);
      b.mean2 = take(c, B); b.rstd2 = take(c, B);
      b.xout = make_buf(c, B, E, 1);
    }
    h->dq = make_buf(c, B, h->hdk, 1); h->dk = make_buf(c, B, h->hdk, 1); h->dv = make_buf(c, B, h->hdk, 1);
    h->d_o = make_buf(c, B, h->hdk, 1);
    h->dz1 = make_buf(c, B, E, 1); h->dz2 = make_buf(c, B, E, 1); h->dh_ff = make_buf(c, B, E, 1);
    h->dxq = make_buf(c, B, E, 1); h->dxk = make_buf(c, B, E, 1); h->dxv = make_buf(c, B, E, 1);
    h->d_ff.assign(nf + 1, Buf());
    for (int j = 1; j <= nf; ++j) h->d_ff[j] = make_buf(c, B, h->ff_arch[j - 1], 1);
    h->pooled = make_buf(c, h->maxSets, E, 1);
    h->d_pooled = make_buf(c, h->maxSets, E, 1);
    if (h->varlen) h->dsum = take(c, h->maxSets * h->heads * h->Ls);
  }
  h->ws_floats = h->plan_floats = c;
}

// the compiled metrics' workspace behind the plan: nothing without metrics
void plan_metrics(dib_model* h) {
  long long c = h->plan_floats;
  if (h->metrics.count > 0) {
    h->metric_z_off = take(c, (h->st ? h->maxSets : h->maxB) * h->out);
    h->metric_part_off = take(c, (long long)kDibMetricMaxCtas * h->metrics.tail);
  }
  h->ws_floats = c;
}

int32_t stats_count(const dib_model* h) { return h->F + 3 + (h->metrics.count > 0 ? h->metrics.tail : 0); }

// a float offset and leading dimension inside the workspace
struct Operand { long long off = 0; int ld = 0; };
Operand opnd(const Buf& b, int g = 0) { return {b.off + g * b.feat_stride, b.ld}; }

// what build_stack asks of group g at boundary k = 0..L+1 of a stack: the input of layer k, the output of layer k-1
struct StackPoint {
  int width = 0;            // columns: layer k's fan-in, layer k-1's fan-out
  Operand in;               // what layer k reads (Dropout's output when there is one)
  Operand act;              // what layer k-1 writes, after its activation and before Dropout: layer k's DGRAD takes act' of it
  Operand grad;             // d (layer k-1's pre-activation output), which layer k's DGRAD writes; k = 0: d (the stack's input)
  long long W = 0, b = 0;   // layer k's kernel [width, next width] and bias
};

// the FWD, DGRAD and WGRAD problems of layers 0..L: the hidden layers apply act, layer L out_act; the DGRAD of layer 0
// (dgrad0) differentiates no activation
template <class At>
Stack build_stack(std::vector<DibGemmProblem>& v, int G, int L, int act, int out_act, bool dgrad0, At at) {
  Stack s;
  s.G = G; s.dgrad0 = dgrad0;
  s.fwd.assign(L + 1, -1); s.dgrad.assign(L + 1, -1); s.wgrad.assign(L + 1, -1);
  s.fan_in.assign(L + 1, 0); s.fan_out.assign(L + 1, 0);
  for (int j = 0; j <= L; ++j) {
    s.fan_out[j] = at(0, j + 1).width;
    for (int g = 0; g < G; ++g)
      if (at(g, j).width > s.fan_in[j]) s.fan_in[j] = at(g, j).width;
  }
  std::vector<int>* first[3] = {&s.fwd, &s.dgrad, &s.wgrad};
  for (int mode = DIB_GEMM_FWD; mode <= DIB_GEMM_WGRAD; ++mode)
    for (int j = mode == DIB_GEMM_DGRAD && !dgrad0 ? 1 : 0; j <= L; ++j) {
      (*first[mode])[j] = (int)v.size();
      for (int g = 0; g < G; ++g) {
        const StackPoint x = at(g, j), y = at(g, j + 1);
        DibGemmProblem p;
        memset(&p, 0, sizeof(p));
        if (mode == DIB_GEMM_FWD) {            // y.act = act(x.in W + b)
          p.a_off = x.in.off; p.lda = x.in.ld; p.b_off = x.W; p.ldb = y.width; p.c_off = y.act.off; p.ldc = y.act.ld;
          p.x_off = x.b; p.T = x.width; p.C = y.width; p.act = j < L ? act : out_act;
        } else if (mode == DIB_GEMM_DGRAD) {   // x.grad = y.grad W^T * act'(x.act)
          p.a_off = y.grad.off; p.lda = y.grad.ld; p.b_off = x.W; p.ldb = y.width; p.c_off = x.grad.off; p.ldc = x.grad.ld;
          if (j > 0) { p.x_off = x.act.off; p.ldx = x.act.ld; }
          p.T = y.width; p.C = x.width; p.act = j > 0 ? act : DIB_ACT_LINEAR;
        } else {                               // dW = x.in^T y.grad, db = column sums of y.grad
          p.a_off = x.in.off; p.lda = x.in.ld; p.b_off = y.grad.off; p.ldb = y.grad.ld; p.c_off = x.W; p.ldc = y.width;
          p.x_off = x.b; p.R = x.width; p.C = y.width;
        }
        v.push_back(p);
      }
    }
  return s;
}

void build_problems(dib_model* h, std::vector<DibGemmProblem>& v) {
  const int L = h->L, Li = h->Li, Ly = h->Ly, E = h->E, hdk = h->hdk, nf = nff(h);
  if (!h->simple) {
    h->enc_stack = build_stack(v, h->F, L, h->act, DIB_ACT_LINEAR, false, [&](int f, int k) {
      StackPoint p;
      if (k > L) { p.width = 2 * E; p.act = opnd(h->enc_out, f); p.grad = opnd(h->d_out, f); return p; }
      p.width = enc_fan_in(h, f, k);
      p.in = k == 0 ? Operand{h->pe.off + h->pe_off[f], h->ldpe} : opnd(h->drop > 0.f ? h->enc_drop[k] : h->enc_act[k], f);
      p.act = opnd(h->enc_act[k], f); p.grad = opnd(h->d_enc[k], f);
      p.W = h->encW[f][k]; p.b = h->encB[f][k];
      return p;
    });
    h->enc_stack.drop = h->drop;
    h->enc_stack.label = "enc";
  }
  h->int_stack = build_stack(v, 1, Li, h->act, h->out_act, true, [&](int, int k) {   // the set transformer's head reads the set means
    StackPoint p;
    if (k > Li) { p.width = h->out; p.act = opnd(h->pred); p.grad = opnd(h->d_pred); return p; }
    p.width = int_fan_in(h, k);
    if (k == 0) { p.in = opnd(h->st ? h->pooled : h->emb); p.grad = opnd(h->st ? h->d_pooled : h->d_emb); }
    else { p.in = p.act = opnd(h->int_act[k]); p.grad = opnd(h->d_int[k]); }
    p.W = h->intW[k]; p.b = h->intB[k];
    return p;
  });
  h->int_stack.label = "int";
  // the dense layers of the attention blocks, all on n * Ls particle rows: Q / K / V as one group of three (same input,
  // kernels [E, h*dk]), the output projection [h*dk, E], the FF stack on LN1's output
  for (int b = 0; b < h->nblk; ++b) {
    dib_model::StBlock& k = h->blk[b];
    const Buf& x = b == 0 ? h->emb : h->blk[b - 1].xout;
    const long long W[3] = {k.Wq, k.Wk, k.Wv}, bias[3] = {k.bq, k.bk, k.bv};
    const Buf* qkv[3] = {&k.q, &k.k, &k.v};
    const Buf* dqkv[3] = {&h->dq, &h->dk, &h->dv};
    const Buf* dx[3] = {&h->dxq, &h->dxk, &h->dxv};
    k.qkv_stack = build_stack(v, 3, 0, DIB_ACT_LINEAR, DIB_ACT_LINEAR, true, [&](int i, int q) {
      StackPoint p;
      if (q == 0) { p.width = E; p.in = opnd(x); p.grad = opnd(*dx[i]); p.W = W[i]; p.b = bias[i]; }
      else { p.width = hdk; p.act = opnd(*qkv[i]); p.grad = opnd(*dqkv[i]); }
      return p;
    });
    k.o_stack = build_stack(v, 1, 0, DIB_ACT_LINEAR, DIB_ACT_LINEAR, true, [&](int, int q) {
      StackPoint p;
      if (q == 0) { p.width = hdk; p.in = opnd(k.o); p.grad = opnd(h->d_o); p.W = k.Wo; p.b = k.bo; }
      else { p.width = E; p.act = opnd(k.a); p.grad = opnd(h->dz1); }
      return p;
    });
    k.ff_stack = build_stack(v, 1, nf - 1, h->ff_act, h->ff_act, true, [&](int, int q) {
      StackPoint p;
      p.width = ff_fan_in(h, q);
      p.in = opnd(q == 0 ? k.hh : k.ff[q]); p.act = opnd(k.ff[q]); p.grad = opnd(q == 0 ? h->dh_ff : h->d_ff[q]);
      if (q < nf) { p.W = k.ffW[q]; p.b = k.ffB[q]; }
      return p;
    });
  }
  if (!infonce(h)) return;
  // the output encoder on its own buffers (train.py:186-193); no gradient is taken with respect to y itself
  h->y_stack = build_stack(v, 1, Ly, h->act, DIB_ACT_LINEAR, false, [&](int, int k) {
    StackPoint p;
    if (k > Ly) { p.width = h->out; p.act = opnd(h->y_out); p.grad = opnd(h->d_y_out); return p; }
    p.width = y_fan_in(h, k);
    p.in = k == 0 ? Operand{h->ype.off, h->ldype} : opnd(h->y_act[k]);
    p.act = opnd(h->y_act[k]); p.grad = opnd(h->d_yact[k]);
    p.W = h->yW[k]; p.b = h->yB[k];
    return p;
  });
  h->y_stack.label = "y";
}

struct Ctx {
  dib_model* h;
  const float* params;
  float* ws;
  cudaStream_t st;
  int n;
  bool dev_step = false;     // dib_train_step only: add *h->step_dev to the Philox step word (dib_set_noise_step_device)
  const uint32_t* step_dev() const { return dev_step ? h->step_dev : nullptr; }
  const int* sizes = nullptr;   // particle-row contexts of a variable-size set transformer: the bound set sizes
};

void prof_begin(const Ctx& c, const char* label, int j = -1) {
  if (!c.h->profiling) return;
  dib_model::ProfRec r;
  r.label = label;
  if (j >= 0) r.label += std::to_string(j);
  cudaEventCreate(&r.a); cudaEventCreate(&r.b);
  cudaEventRecord(r.a, c.st);
  c.h->prof.push_back(r);
}
void prof_end(const Ctx& c) {
  if (!c.h->profiling) return;
  cudaEventRecord(c.h->prof.back().b, c.st);
}

int gemm(const Ctx& c, int mode, int first, int nprob, int maxC, int maxR, int nsplit, int rps) {
  DibGemmLaunch L;
  L.probs = c.h->d_probs + first;
  L.nprob = nprob;
  L.M = c.n;
  L.maxC = maxC; L.maxR = maxR;
  L.nsplit = nsplit; L.rows_per_split = rps; L.split_stride = c.h->Pp;
  L.alpha = c.h->alpha;
  float* part = c.ws + c.h->part_off;
  const bool tc = is_tc(c.h);
  L.round_out = tc ? 1 : 0;
  switch (mode) {
    case DIB_GEMM_FWD: L.baseA = c.ws; L.baseB = c.params; L.baseC = c.ws; L.baseX = nullptr; break;
    case DIB_GEMM_DGRAD: L.baseA = c.ws; L.baseB = c.params; L.baseC = c.ws; L.baseX = c.ws; break;
    default: L.baseA = c.ws; L.baseB = c.ws; L.baseC = part; L.baseX = part; break;
  }
  if (tc && dib_gemm_tc_eligible(mode, c.h->h_probs.data() + first, nprob, c.params)) {
    if (mode != DIB_GEMM_WGRAD) { L.baseB = c.ws + c.h->wshadow_off; L.baseBias = c.params; }
    DIB_CUDA_OK(dib_launch_gemm_tc(mode, L, c.h->h_probs.data() + first, c.st));
    return 0;
  }
  DIB_CUDA_OK(dib_launch_gemm_simt(mode, L, c.st));
  return 0;
}

int check_call(const dib_model* h, const void* params, const void* x, int64_t n, const void* ws) {
  if (!h) return fail("null model handle");
  if (!params || !ws || (!x && n > 0)) return fail("null params / x / workspace pointer");
  if (n < 0 || n > h->maxB) return fail("n = " + std::to_string(n) + " exceeds config.max_batch = " + std::to_string(h->maxB));
  if (reinterpret_cast<uintptr_t>(ws) & 255) return fail("workspace must be 256-byte aligned");
  if (reinterpret_cast<uintptr_t>(params) & 15) return fail("params must be 16-byte aligned");
  return 0;
}

// calls whose n counts sets on a set-transformer handle (check_call bounds particle rows)
int check_sets(const dib_model* h, int64_t n) {
  if (h->st && n > h->maxSets)
    return fail("n = " + std::to_string(n) + " sets exceeds config.max_batch = " + std::to_string(h->maxSets));
  if (h->varlen && n > 0 && !h->set_sizes_dev)
    return fail("variable set sizes: bind the sizes of the n sets with dib_set_set_sizes_device before this call");
  return 0;
}

// noise of one forward: the caller's eps, or Philox (seed, step, sample_offset); training turns Dropout on
struct NoiseKey { const float* eps; uint64_t seed; uint32_t step; uint64_t sample_offset; bool training; };

// the encoder side of a call on n sets: the encoders and the attention blocks run on its n * Ls particle rows (with the bound
// sizes of a variable-size model), their noise keyed by the global particle row.  An MLP model (Ls = 1, no sizes) gets the call
// unchanged.
struct RowView { Ctx c; NoiseKey nk; };
RowView particle_rows(const Ctx& c, const NoiseKey& nk) {
  const dib_model* h = c.h;
  RowView r{c, nk};
  r.c.n = c.n * h->Ls;
  r.c.sizes = h->varlen ? h->set_sizes_dev : nullptr;
  r.nk.sample_offset = nk.sample_offset * (uint64_t)h->Ls;
  return r;
}

int encode_all(const Ctx& c, const float* x, int ldx, int feature, const int* row_index, int64_t n_src, const NoiseKey* key = nullptr);

// TF32 GEMMs read the weights through a TF32-rounded copy
int tf32_shadow(const Ctx& c) {
  if (!is_tc(c.h)) return 0;
  prof_begin(c, "weights_tf32_shadow");
  DIB_CUDA_OK(dib_launch_round_copy(c.params, c.ws + c.h->wshadow_off, c.h->P, c.st));
  prof_end(c);
  return 0;
}

// FWD of layers 0..L of `groups` groups from `first` (all, or one feature of the encoders).  Dropout (the encoders) runs after
// each hidden layer: keyed by `key` in training, the identity copy otherwise.
int stack_forward(const Ctx& c, const Stack& s, int first, int groups, const NoiseKey* key = nullptr) {
  dib_model* h = c.h;
  const int L = (int)s.fwd.size() - 1;
  const bool tr = key && key->training;
  for (int j = 0; j <= L; ++j) {
    if (s.label) prof_begin(c, (std::string(s.label) + "_fwd_l").c_str(), j);
    if (gemm(c, DIB_GEMM_FWD, s.fwd[j] + first, groups, s.fan_out[j], 0, 1, 0)) return 1;
    if (j < L && s.drop > 0.f) {
      const Buf& a = h->enc_act[j + 1];
      DIB_CUDA_OK(dib_launch_dropout(c.ws + a.off, c.ws + h->enc_drop[j + 1].off, a.feat_stride, a.ld, s.fan_out[j], s.G, c.n,
                                     tr ? s.drop : 0.f, key ? key->seed : 0, key ? key->step : 0, tr ? c.step_dev() : nullptr,
                                     key ? key->sample_offset : 0, j + 1, groups < s.G ? first : -1, 0, is_tc(h) ? 1 : 0, c.st));
    }
    if (s.label) prof_end(c);
  }
  return 0;
}

// for j = L..0: WGRAD of layer j into the split-partial table, then its DGRAD (layer 0: with dgrad0) and Dropout's backward
// (the same keep mask as the training forward keyed by `key`, scaled)
int stack_backward(const Ctx& c, const Stack& s, const Split& sp, const NoiseKey* key = nullptr) {
  dib_model* h = c.h;
  for (int j = (int)s.fwd.size() - 1; j >= 0; --j) {
    if (s.label) prof_begin(c, (std::string(s.label) + "_wgrad_l").c_str(), j);
    if (gemm(c, DIB_GEMM_WGRAD, s.wgrad[j], s.G, s.fan_out[j], s.fan_in[j], sp.nsplit, (int)sp.rps)) return 1;
    if (s.label) prof_end(c);
    if (j == 0 && !s.dgrad0) continue;
    if (s.label) prof_begin(c, (std::string(s.label) + "_dgrad_l").c_str(), j);
    if (gemm(c, DIB_GEMM_DGRAD, s.dgrad[j], s.G, s.fan_in[j], 0, 1, 0)) return 1;
    if (s.drop > 0.f) {
      const Buf& d = h->d_enc[j];
      DIB_CUDA_OK(dib_launch_dropout(nullptr, c.ws + d.off, d.feat_stride, d.ld, s.fan_in[j], s.G, c.n, s.drop, key->seed, key->step,
                                     c.step_dev(), key->sample_offset, j, -1, 1, is_tc(h) ? 1 : 0, c.st));
    }
    if (s.label) prof_end(c);
  }
  return 0;
}

DibReparamArgs reparam_args(const Ctx& c, const NoiseKey& nk) {
  const dib_model* h = c.h;
  DibReparamArgs ra;
  ra.enc_out = c.ws + h->enc_out.off; ra.feat_stride = h->enc_out.feat_stride; ra.ldo = h->enc_out.ld;
  ra.eps = nk.eps; ra.seed = nk.seed; ra.step = nk.step; ra.step_dev = c.step_dev(); ra.sample_offset = nk.sample_offset;
  ra.F = h->F; ra.E = h->E; ra.n = c.n; ra.round_out = is_tc(h) ? 1 : 0;
  ra.set_sizes = c.sizes; ra.set_len = h->Ls;
  return ra;
}

// inputs of the fused encoder kernels; the forward adds its outputs
DibEncFusedIO fused_io(const Ctx& c, const float* x, const NoiseKey& nk) {
  DibEncFusedIO io;
  io.params = c.params; io.packed = c.ws + c.h->pack_off; io.x = x; io.ldx = c.h->D; io.n = c.n;
  io.eps = nk.eps; io.seed = nk.seed; io.step = nk.step; io.step_dev = c.step_dev(); io.sample_offset = nk.sample_offset;
  io.emb = nullptr; io.ldemb = 0; io.user_emb = nullptr; io.kl_part = nullptr; io.kl_stride = 0;
  return io;
}

// 16-bit activation entering integration layer j
const void* int16_in(const Ctx& c, int j) {
  return j == 0 ? (const void*)(c.ws + c.h->emb16_off) : (const void*)(c.ws + c.h->g16_off[j]);
}

// encoder half of the forward: PE -> encoder layers (all features) -> reparam / KL partials.  Writes the embedding the
// integration half reads (fp32 workspace copy, or the fp16 copy of the 16-bit integration network; neither when enc_only:
// the caller's network consumes user_emb) and *nblk_kl = KL partials per feature.
int forward_encoders(const Ctx& c, const float* x, const NoiseKey& nk, float* user_emb, bool enc_only, int* nblk_kl) {
  dib_model* h = c.h;
  if (!h->route.enc_fused) {
    if (encode_all(c, x, h->D, -1, nullptr, 0, &nk)) return 1;
    prof_begin(c, "reparam_kl_fwd");
    DIB_CUDA_OK(dib_launch_reparam_fwd(reparam_args(c, nk), c.ws + h->emb.off, h->emb.ld, user_emb, c.ws + h->kl_part_off,
                                       h->kl_stride, c.st));
    prof_end(c);
    *nblk_kl = (int)DIB_CEIL_DIV((long long)c.n, (long long)kRowsPerBlock);
    return 0;
  }
  const long long want = (long long)h->F * DIB_CEIL_DIV((long long)c.n, 128ll);
  const long long cap = (long long)h->num_sms * dib_enc_fused_fwd_ctas_per_sm();
  DibEncFusedDesc d = h->fdesc;
  d.logvar_offset = h->lv_off;
  d.grid = (int)(want < cap ? want : cap);
  *nblk_kl = DIB_CEIL_DIV(d.grid, h->F);
  prof_begin(c, "enc_pack_weights");
  {
    const long long zn = (long long)h->F * h->kl_stride, zcap = dib_enc_fused_pack_zero_capacity(h->F);
    // the pack kernel also clears the KL partial table when it fits its grid
    if (zn <= zcap) DIB_CUDA_OK(dib_enc_fused_pack(d, c.params, c.ws + h->pack_off, c.ws + h->kl_part_off, zn, c.st));
    else {
      DIB_CUDA_OK(dib_enc_fused_pack(d, c.params, c.ws + h->pack_off, nullptr, 0, c.st));
      DIB_CUDA_OK(cudaMemsetAsync(c.ws + h->kl_part_off, 0, sizeof(float) * (size_t)zn, c.st));
    }
  }
  prof_end(c);
  const bool i16 = h->route.int16 && !enc_only;
  DibEncFusedIO io = fused_io(c, x, nk);
  io.emb = i16 || enc_only ? nullptr : c.ws + h->emb.off; io.ldemb = h->emb.ld; io.user_emb = user_emb;
  io.kl_part = c.ws + h->kl_part_off; io.kl_stride = h->kl_stride;
  if (i16) { io.emb16 = c.ws + h->emb16_off; io.ldemb16 = h->F * h->E; }
  prof_begin(c, "enc_fused_fwd");
  DIB_CUDA_OK(dib_enc_fused_forward(d, io, c.st));
  prof_end(c);
  return 0;
}

// e2 = output_encoder(y) into y_out (train.py:186-193)
int forward_output_encoder(const Ctx& c, const float* y) {
  dib_model* h = c.h;
  prof_begin(c, "y_pe");
  DIB_CUDA_OK(dib_launch_pe(y, h->ydim, 0, h->d_ycol_src, h->d_ycol_freq, 0, h->ldype, c.ws + h->ype.off, h->ldype, 0, c.n,
                            is_tc(h) ? 1 : 0, c.st));
  prof_end(c);
  return stack_forward(c, h->y_stack, 0, 1);
}

// the streaming InfoNCE of the c.n own rows [row0, row0 + c.n) of e1 / e2 [n, d] against all n rows: r and c at lse_stride,
// s_ii, the loss sum and the accuracy zero in the workspace; d loss / d e1 into d_pred (what the DIB_LOSS_EXTERNAL backward
// reads) and d loss / d e2 into d_y_out (what backward_output_encoder reads), both at local row index
DibInfonceStream infonce_args(const Ctx& c, const float* e1, int ld1, const float* e2, int ld2, long long n, long long row0,
                              float* lse_r, float* lse_c, int lse_stride) {
  const dib_model* h = c.h;
  DibInfonceStream a;
  a.kind = h->sim_kind; a.temperature = h->temperature;
  a.e1 = e1; a.ld1 = ld1;
  a.e2 = e2; a.ld2 = ld2;
  a.n = n; a.d = h->out;
  a.row0 = row0; a.rows = c.n;
  a.lse_r = lse_r; a.lse_c = lse_c; a.lse_stride = lse_stride;
  a.diag = c.ws + h->nce_off + 2 * (long long)c.n;
  a.loss_sum = c.ws + h->loss_part_off; a.acc_zero = c.ws + h->acc_part_off;
  a.d_e1 = c.ws + h->d_pred.off; a.ld_d1 = h->d_pred.ld;
  a.d_e2 = c.ws + h->d_y_out.off; a.ld_d2 = h->d_y_out.ld;
  a.round_out = is_tc(h) ? 1 : 0;
  return a;
}

// the row / column sweeps and the loss sum of the own rows, then the stats row (KL sums of the forward, n = own rows)
int infonce_loss_stats(const Ctx& c, const DibInfonceStream& a, float* out_stats, int nblk_kl) {
  dib_model* h = c.h;
  prof_begin(c, "infonce_loss_stats");
  DIB_CUDA_OK(dib_launch_infonce_stream_loss(a, c.st));
  DIB_CUDA_OK(dib_launch_finalize_stats(c.ws + h->kl_part_off, h->kl_stride, nblk_kl, c.ws + h->loss_part_off, c.ws + h->acc_part_off,
                                        1, h->F, c.n, 1, out_stats, c.st));
  prof_end(c);
  return 0;
}

int infonce_grads(const Ctx& c, const DibInfonceStream& a) {
  prof_begin(c, "infonce_grads");
  DIB_CUDA_OK(dib_launch_infonce_stream_grads(a, c.st));
  prof_end(c);
  return 0;
}

// DIB_LOSS_INFONCE with targets on one GPU, after the integration network wrote e1 = pred: output encoder e2 = output_encoder(y),
// the streaming InfoNCE loss over all c.n rows into the stats row and, training, its gradients
int forward_infonce(const Ctx& c, const float* y, bool training, float* user_pred, float* out_stats, int nblk_kl) {
  dib_model* h = c.h;
  if (forward_output_encoder(c, y)) return 1;
  float* scratch = c.ws + h->nce_off;
  const DibInfonceStream a = infonce_args(c, c.ws + h->pred.off, h->pred.ld, c.ws + h->y_out.off, h->y_out.ld, c.n, 0, scratch,
                                          scratch + c.n, 1);
  if (infonce_loss_stats(c, a, out_stats, nblk_kl)) return 1;
  if (user_pred) DIB_CUDA_OK(dib_launch_copy2d(c.ws + h->pred.off, h->pred.ld, user_pred, h->out, h->out, c.n, c.st));
  if (training && infonce_grads(c, a)) return 1;
  return 0;
}

// integration half of the forward: integration layers -> prediction, compiled loss / metrics, d loss / d prediction
// (training) -> the stats row
int forward_loss(const Ctx& c, const float* y, float inv_batch, bool training, float* user_pred, float* out_stats,
                 int nblk_kl) {
  dib_model* h = c.h;
  const float* weights = y ? h->sample_weights_dev : nullptr;
  auto finalize = [&](int nblk_loss) {
    return dib_launch_finalize_stats(c.ws + h->kl_part_off, h->kl_stride, nblk_kl, c.ws + h->loss_part_off, c.ws + h->acc_part_off,
                                     nblk_loss, h->F, c.n, y != nullptr, out_stats, c.st);
  };
  if (!h->route.int16) {
    if (stack_forward(c, h->int_stack, 0, 1)) return 1;
    if (infonce(h) && y) return forward_infonce(c, y, training, user_pred, out_stats, nblk_kl);
    prof_begin(c, "loss_stats");
    DIB_CUDA_OK(dib_launch_loss(h->loss, h->out_act, h->alpha, c.ws + h->pred.off, h->pred.ld, y, h->out, c.n, inv_batch,
                                training ? c.ws + h->d_pred.off : nullptr, user_pred, c.ws + h->loss_part_off,
                                c.ws + h->acc_part_off, is_tc(h) ? 1 : 0, weights, c.st));
    DIB_CUDA_OK(finalize((int)DIB_CEIL_DIV((long long)c.n, (long long)kRowsPerBlock)));
    prof_end(c);
    return 0;
  }
  // ---------------- integration network on 16-bit activations + fused output head
  const int bf = h->precision == DIB_PREC_BF16 ? 1 : 0;
  prof_begin(c, "int16_pack_weights");
  {
    std::vector<const float*> wsrc; std::vector<void*> wdst; std::vector<long long> wn;
    for (int j = 0; j < h->Li; ++j) {
      wsrc.push_back(c.params + h->intW[j]); wdst.push_back(c.ws + h->w16_off[j]);
      wn.push_back((long long)int_fan_in(h, j) * int_fan_out(h, j));
    }
    DIB_CUDA_OK(dib_int16_convert_many(wsrc.data(), wdst.data(), wn.data(), h->Li, bf, c.st));
  }
  prof_end(c);
  const float gscale = training ? loss_scale(inv_batch) : 1.f;
  void* const dg = training ? (void*)(c.ws + h->dg16_off[h->Li]) : nullptr;
  const int n_plain = h->route.tail_fused ? h->Li - 2 : h->Li;
  for (int j = 0; j < n_plain; ++j) {
    prof_begin(c, "int16_fwd_l", j);
    DIB_CUDA_OK(dib_int16_fwd(int16_in(c, j), int_fan_in(h, j), c.ws + h->w16_off[j], c.params + h->intB[j], c.ws + h->g16_off[j + 1],
                              int_fan_out(h, j), c.n, int_fan_in(h, j), int_fan_out(h, j), h->act, h->alpha, bf, c.st));
    prof_end(c);
  }
  if (h->route.tail_fused) {
    // the last two hidden layers and the head run as ONE kernel (g2 stays on chip); in training on the tail_bwd route it
    // continues with the dgrad chain (dg1 -> dg16_off[j1], its column sums -> the dbpart row of layer j1, and d emb when
    // j0 == 0) that backward_integration then skips
    const int j0 = h->Li - 2, j1 = h->Li - 1;
    const bool bwd = training && h->route.tail_bwd;
    prof_begin(c, bwd ? "int16_fwd2_head_dgrad" : "int16_fwd2_head");
    DIB_CUDA_OK(dib_int16_fwd2_head(int16_in(c, j0), int_fan_in(h, j0), int_fan_in(h, j0), c.ws + h->w16_off[j0], c.params + h->intB[j0],
                                    c.ws + h->w16_off[j1], c.params + h->intB[j1], c.ws + h->g16_off[j1], c.params + h->intW[h->Li],
                                    c.params + h->intB[h->Li], h->act, h->out_act, h->alpha, h->loss, y, c.n, inv_batch, gscale, dg,
                                    bwd ? (void*)(c.ws + h->dg16_off[j1]) : nullptr,
                                    bwd ? c.ws + h->dbpart_off + (long long)j1 * h->dbpart_layer : nullptr,
                                    bwd && j0 == 0 ? (void*)(c.ws + h->demb16_off) : nullptr, user_pred, c.ws + h->headpart_off,
                                    h->head_stride, c.ws + h->loss_part_off, c.ws + h->acc_part_off, &h->head_used, weights, bf,
                                    c.st));
    DIB_CUDA_OK(finalize(h->head_used));
    prof_end(c);
    return 0;
  }
  const int Kh = h->int_arch[h->Li - 1];
  h->head_used = h->head_blocks;
  prof_begin(c, "int16_head_loss");
  DIB_CUDA_OK(dib_int16_head(c.ws + h->g16_off[h->Li], Kh, Kh, c.params + h->intW[h->Li], c.params + h->intB[h->Li], h->out,
                             h->out_act, h->act, h->alpha, h->loss, y, c.n, inv_batch, gscale, dg, Kh, user_pred, c.ws + h->headpart_off,
                             h->head_stride, c.ws + h->loss_part_off, c.ws + h->acc_part_off, h->head_blocks, h->route.head1, weights,
                             bf, c.st));
  DIB_CUDA_OK(finalize(h->head_blocks));
  prof_end(c);
  return 0;
}

// every feature encoder (feature = -1), or feature `feature` alone reading only its columns of x, on n rows of x
// (deterministic part: mu | logvar incl. the offset) into the enc_out workspace buffer: positional encoding + grouped GEMMs
// (models.py:72-78,106), or nb-bool's SimpleEncoder constants
int encode_all(const Ctx& c, const float* x, int ldx, int feature, const int* row_index, int64_t n_src, const NoiseKey* key) {
  dib_model* h = c.h;
  const int f = feature;
  if (h->simple) {
    prof_begin(c, "simple_enc_fwd");
    DIB_CUDA_OK(dib_launch_simple_enc_fwd(x, ldx, h->d_xoff, c.params, c.ws + h->enc_out.off, h->enc_out.feat_stride,
                                          h->enc_out.ld, h->F, h->E, c.n, f, f >= 0 ? 1 : 0, row_index, n_src, c.st));
    prof_end(c);
  } else {
    prof_begin(c, "pe");
    DIB_CUDA_OK(dib_launch_pe(x, ldx, f >= 0 ? h->x_off[f] : 0, h->d_col_src, h->d_col_freq, f >= 0 ? h->pe_off[f] : 0,
                              f >= 0 ? h->pe_off[f] + DIB_ROUND_UP(h->w_in[f], 4) : h->ldpe, c.ws + h->pe.off, h->ldpe, 0, c.n,
                              is_tc(h) ? 1 : 0, c.st, row_index, row_index ? h->d_col_feat : nullptr, n_src));
    // padding particles enter the first layer as zeros: whatever x holds there, every activation of theirs stays finite
    if (c.sizes) DIB_CUDA_OK(dib_launch_zero_pad_rows(c.ws + h->pe.off, h->ldpe, c.n, h->Ls, c.sizes, c.st));
    prof_end(c);
    if (stack_forward(c, h->enc_stack, f >= 0 ? f : 0, f >= 0 ? 1 : h->F, key)) return 1;
  }
  DIB_CUDA_OK(dib_launch_add_logvar_offset(c.ws + h->enc_out.off, h->enc_out.feat_stride, h->enc_out.ld, h->F, h->E, c.n,
                                           h->lv_off, f, c.st));
  return 0;
}

// weight for the per-sample KL gradients: beta itself (models.py:118) or d(beta*scale*KL^p)/dKL (nb-chaos cell 10)
int ib_weight(const Ctx& c, const float* beta_dev, const float* stats, float inv_global_batch, const float** out) {
  dib_model* h = c.h;
  *out = beta_dev;
  if (h->kl_exp == 1.f && h->kl_scale == 1.f) return 0;
  float* be = c.ws + h->beta_eff_off;
  DIB_CUDA_OK(dib_launch_beta_eff(stats, h->F, inv_global_batch, beta_dev, h->kl_exp, h->kl_scale, be, c.st));
  *out = be;
  return 0;
}

// encoder backward from d emb -- fp32 (d_emb, ldd) or the fp16 copy the 16-bit integration backward leaves, already x the loss
// scale (d_emb16) -- into the split-partial table: the encoder parameters' weight-gradient partials in rows [0, *nrows).
// Relies on the workspace as the forward of the same (x, noise) left it.
int backward_encoders(const Ctx& c, const float* x, const NoiseKey& nk, const float* d_emb, int ldd, const void* d_emb16,
                      const float* beta_w, float inv_batch, const Split& sp, int* nrows) {
  dib_model* h = c.h;
  float* part = c.ws + h->part_off;
  if (h->route.enc_fused) {
    const long long p_enc = h->intW[0];
    const long long want = (long long)h->F * DIB_CEIL_DIV((long long)c.n, 128ll);
    DibEncFusedDesc d = h->fdesc;
    d.grid = (int)(want < h->num_sms ? want : h->num_sms);
    const int slots_max = DIB_CEIL_DIV(d.grid, h->F), slots_min = d.grid / h->F;
    // features served by one CTA fewer leave their last slot unwritten: zero it (ENCODER range only -- the
    // integration network's batch-split partials live in the same rows beyond p_enc)
    for (int srow = slots_min; srow < slots_max; ++srow)
      DIB_CUDA_OK(cudaMemsetAsync(part + (long long)srow * h->Pp, 0, sizeof(float) * (size_t)p_enc, c.st));
    DibEncFusedBwdIO b;
    b.d_emb = d_emb; b.ldd = ldd; b.d_emb16 = d_emb16; b.ldd16 = d_emb16 ? h->F * h->E : 0;
    b.beta_dev = beta_w; b.inv_batch = inv_batch; b.gscale = loss_scale(inv_batch); b.part = part; b.split_stride = h->Pp;
    prof_begin(c, "enc_fused_bwd");
    DIB_CUDA_OK(dib_enc_fused_backward(d, fused_io(c, x, nk), b, c.st));
    prof_end(c);
    *nrows = slots_max;
    return 0;
  }
  prof_begin(c, "reparam_kl_bwd");
  DIB_CUDA_OK(dib_launch_reparam_bwd(reparam_args(c, nk), d_emb, ldd, beta_w, inv_batch, c.ws + h->d_out.off, c.st));
  prof_end(c);
  if (h->simple) {
    prof_begin(c, "simple_enc_wgrad");
    DIB_CUDA_OK(dib_launch_simple_enc_wgrad(x, h->D, h->d_xoff, c.ws + h->d_out.off, h->d_out.feat_stride, h->d_out.ld, h->F, h->E,
                                            c.n, sp.nsplit, (int)sp.rps, part, h->Pp, c.st));
    prof_end(c);
  } else if (stack_backward(c, h->enc_stack, sp, &nk)) {
    return 1;
  }
  *nrows = sp.nsplit;
  return 0;
}

// integration network backward (GradientTape through models.py:122) from d loss / d prediction, as the forward of the step left
// it, down to the d emb backward_encoders reads.  16-bit route: its fixed-order reductions (bias gradients from the head / dgrad
// column sums, batch-split weight-gradient partials, the output layer's per-CTA partials) are appended to *segs for the caller to
// run in one launch with the encoder segment (the 16-bit route implies the fused encoders).  Per-layer GEMM route:
// grads_flat[p_enc, P) is final on return.
int backward_integration(const Ctx& c, float inv_batch, const Split& sp, float* grads_flat, std::vector<DibReduceSeg>* segs) {
  dib_model* h = c.h;
  float* part = c.ws + h->part_off;
  if (!h->route.int16) {
    const long long p_enc = h->intW[0];
    if (stack_backward(c, h->int_stack, sp)) return 1;
    prof_begin(c, "int_split_reduce");
    DIB_CUDA_OK(dib_launch_reduce_partials(part + p_enc, h->Pp, sp.nsplit, h->Px - p_enc, grads_flat + p_enc, c.st));
    prof_end(c);
    return 0;
  }
  const int bf = h->precision == DIB_PREC_BF16 ? 1 : 0;
  const float gscale = loss_scale(inv_batch);
  const int Kh = h->int_arch[h->Li - 1];
  const int row_tiles = (int)DIB_CEIL_DIV((long long)c.n, 128ll);
  const long long p_head = h->intW[h->Li];
  // bias gradient of the last hidden layer: column sums of dg accumulated by the output head
  segs->push_back({c.ws + h->headpart_off + (long long)Kh * h->out + h->out, h->head_stride, h->head_used, Kh, 1.f / gscale,
                   grads_flat + h->intB[h->Li - 1]});
  // the dgrad chain first (layer j's dgrad produces the gradient layer j-1's wgrad consumes), then the weight gradients in PAIRS of
  // layers per launch: one layer's [K/128 x N/128 x splits] tiles do not fill the 2 x SMs CTA slots, two layers' tiles do.
  // On the tail_bwd route the training forward already ran the dgrads of layer j1 = Li-1 and, when j0 = Li-2 is 0, of j0.
  const int j_top = h->route.tail_bwd ? (h->Li == 2 ? -1 : h->Li - 2) : h->Li - 1;
  for (int j = h->Li - 1; j >= 0; --j) {
    const int K = int_fan_in(h, j), N = int_fan_out(h, j);
    if (j <= j_top) {
      prof_begin(c, "int16_dgrad_l", j);
      DIB_CUDA_OK(dib_int16_dgrad(c.ws + h->dg16_off[j + 1], N, c.ws + h->w16_off[j], j > 0 ? (const void*)(c.ws + h->g16_off[j]) : nullptr,
                                  K, j > 0 ? (void*)(c.ws + h->dg16_off[j]) : (void*)(c.ws + h->demb16_off), K, c.n, K, N, h->act,
                                  h->alpha, j > 0 ? c.ws + h->dbpart_off + (long long)j * h->dbpart_layer : nullptr, bf, c.st));
      prof_end(c);
    }
    if (j > 0)   // bias gradient of layer j-1 = column sums of the gradient layer j's dgrad produced
      segs->push_back({c.ws + h->dbpart_off + (long long)j * h->dbpart_layer, K, row_tiles, K, 1.f / gscale, grads_flat + h->intB[j - 1]});
  }
  std::vector<int> nsplit_of(h->Li, sp.nsplit);
  auto tiles_of = [&](int j) { return DIB_CEIL_DIV(int_fan_in(h, j), 128) * DIB_CEIL_DIV(int_fan_out(h, j), 128); };
  auto wgrad_of = [&](int j, int nsplit, int rps) {
    return DibInt16Wgrad{int16_in(c, j), int_fan_in(h, j), c.ws + h->dg16_off[j + 1], int_fan_out(h, j), part + h->intW[j], nsplit, rps};
  };
  int j = h->Li - 1;
  for (; j >= 1; j -= 2) {          // layers (j, j-1) together
    long long ns = (2ll * h->num_sms) / (tiles_of(j) + tiles_of(j - 1));
    if (ns > h->part_rows) ns = h->part_rows;
    if (ns > (long long)c.n / 256) ns = (long long)c.n / 256;
    if (ns < 1) ns = 1;
    const long long rps2 = DIB_ROUND_UP(DIB_CEIL_DIV((long long)c.n, ns), 64);
    const int ns2 = (int)DIB_CEIL_DIV((long long)c.n, rps2);
    nsplit_of[j] = nsplit_of[j - 1] = ns2;
    const DibInt16Wgrad pair[2] = {wgrad_of(j, ns2, (int)rps2), wgrad_of(j - 1, ns2, (int)rps2)};
    prof_begin(c, "int16_wgrad_pair_l", j - 1);
    DIB_CUDA_OK(dib_int16_wgrad(pair, 2, c.n, h->Pp, 1.f / gscale, bf, c.st));
    prof_end(c);
  }
  if (j == 0) {                     // an odd layer count leaves layer 0 alone
    const DibInt16Wgrad l0 = wgrad_of(0, sp.nsplit, (int)sp.rps);
    prof_begin(c, "int16_wgrad_l", 0);
    DIB_CUDA_OK(dib_int16_wgrad(&l0, 1, c.n, h->Pp, 1.f / gscale, bf, c.st));
    prof_end(c);
  }
  // an empty range: these reductions run in the caller's one launch, timed under enc_split_reduce
  prof_begin(c, "int_split_reduce");
  for (int q = 0; q < h->Li; ++q)     // hidden-layer kernels: batch-split partials
    segs->push_back({part + h->intW[q], h->Pp, nsplit_of[q], (long long)int_fan_in(h, q) * int_fan_out(h, q), 1.f, grads_flat + h->intW[q]});
  segs->push_back({c.ws + h->headpart_off, h->head_stride, h->head_used, h->Px - p_head, 1.f, grads_flat + p_head});
  prof_end(c);
  return 0;
}

// the output encoder's backward from the d loss / d e2 forward_infonce left, into grads_flat[Px, P)
int backward_output_encoder(const Ctx& c, const Split& sp, float* grads_flat) {
  dib_model* h = c.h;
  if (stack_backward(c, h->y_stack, sp)) return 1;
  prof_begin(c, "y_split_reduce");
  DIB_CUDA_OK(dib_launch_reduce_partials(c.ws + h->part_off + h->Px, h->Pp, sp.nsplit, h->P - h->Px, grads_flat + h->Px, c.st));
  prof_end(c);
  return 0;
}

// ---- DIB_INTEGRATION_SET_TRANSFORMER: c.n = particle rows (sets * Ls) -----------------------------------------------
DibAttnArgs attn_args(const Ctx& c, const dib_model::StBlock& k) {
  const dib_model* h = c.h;
  DibAttnArgs a;
  a.q = c.ws + k.q.off; a.k = c.ws + k.k.off; a.v = c.ws + k.v.off; a.ld = k.q.ld;
  a.o = c.ws + k.o.off; a.lse = c.ws + k.lse;
  a.sets = c.n / h->Ls; a.heads = h->heads; a.L = h->Ls; a.dk = h->dkey;
  a.round_out = is_tc(h) ? 1 : 0;
  a.dout = c.ws + h->d_o.off; a.dq = c.ws + h->dq.off; a.dk_ = c.ws + h->dk.off; a.dv = c.ws + h->dv.off;
  a.set_sizes = c.sizes; a.dsum = h->varlen ? c.ws + h->dsum : nullptr;
  return a;
}

DibLayerNorm ln_args(const Ctx& c, const Buf& a, const Buf& b, long long gamma, long long beta, const Buf& y, long long mean,
                     long long rstd) {
  DibLayerNorm l;
  l.a = c.ws + a.off; l.b = c.ws + b.off; l.ld = a.ld; l.rows = c.n; l.E = c.h->E;
  l.gamma = c.params + gamma; l.beta = c.params + beta; l.epsilon = c.h->ln_eps;
  l.y = c.ws + y.off; l.mean = c.ws + mean; l.rstd = c.ws + rstd;
  l.round_out = is_tc(c.h) ? 1 : 0;
  return l;
}

// the attention blocks from the embeddings in h->emb, then the mean over each set's particles into h->pooled
int forward_set_blocks(const Ctx& c) {
  dib_model* h = c.h;
  for (int b = 0; b < h->nblk; ++b) {
    const dib_model::StBlock& k = h->blk[b];
    const Buf& x = b == 0 ? h->emb : h->blk[b - 1].xout;
    prof_begin(c, "st_qkv_fwd_b", b);
    if (stack_forward(c, k.qkv_stack, 0, 3)) return 1;
    prof_end(c);
    prof_begin(c, "st_attn_fwd_b", b);
    DIB_CUDA_OK(h->varlen ? dib_launch_attn_varlen_fwd(attn_args(c, k), c.st) : dib_launch_attn_fwd(attn_args(c, k), c.st));
    prof_end(c);
    prof_begin(c, "st_out_proj_ln1_fwd_b", b);
    if (stack_forward(c, k.o_stack, 0, 1)) return 1;
    DIB_CUDA_OK(dib_launch_ln_fwd(ln_args(c, x, k.a, k.g1, k.be1, k.hh, k.mean1, k.rstd1), c.st));
    prof_end(c);
    prof_begin(c, "st_ff_ln2_fwd_b", b);
    if (stack_forward(c, k.ff_stack, 0, 1)) return 1;
    DIB_CUDA_OK(dib_launch_ln_fwd(ln_args(c, k.hh, k.ff[nff(h)], k.g2, k.be2, k.xout, k.mean2, k.rstd2), c.st));
    prof_end(c);
  }
  const Buf& last = h->nblk ? h->blk[h->nblk - 1].xout : h->emb;
  prof_begin(c, "st_pool_fwd");
  if (h->varlen)
    DIB_CUDA_OK(dib_launch_pool_varlen_fwd(c.ws + last.off, last.ld, h->E, h->Ls, c.n / h->Ls, c.sizes, c.ws + h->pooled.off,
                                           h->pooled.ld, is_tc(h) ? 1 : 0, c.st));
  else
    DIB_CUDA_OK(dib_launch_pool_fwd(c.ws + last.off, last.ld, h->E, h->Ls, c.n / h->Ls, c.ws + h->pooled.off, h->pooled.ld,
                                    is_tc(h) ? 1 : 0, c.st));
  prof_end(c);
  return 0;
}

// the blocks' backward from d pooled (the head's DGRAD output) down to d emb, the blocks' weight-gradient and LayerNorm partials
// in rows [0, sp.nsplit) of the split table
int backward_set_blocks(const Ctx& c, const Split& sp) {
  dib_model* h = c.h;
  const int nf = nff(h);
  float* part = c.ws + h->part_off;
  auto ln_bwd = [&](const DibLayerNorm& l, const float* const dy[4], const float* dy_pool, const Buf& d_res, const Buf* d_branch,
                    long long g, long long be) {
    DibLayerNormBwd b;
    for (int q = 0; q < 4; ++q) b.dy[q] = dy[q];
    b.dy_pool = dy_pool; b.pool_rows = h->Ls; b.pool_scale = 1.f / (float)h->Ls; b.set_sizes = c.sizes;
    b.d_res = c.ws + d_res.off; b.d_branch = d_branch ? c.ws + d_branch->off : nullptr; b.branch_act = h->ff_act; b.alpha = h->alpha;
    b.part = part; b.split_stride = h->Pp; b.gamma_off = g; b.beta_off = be; b.nsplit = sp.nsplit; b.rows_per_split = sp.rps;
    return dib_launch_ln_bwd(l, b, c.st);
  };
  for (int b = h->nblk - 1; b >= 0; --b) {
    const dib_model::StBlock& k = h->blk[b];
    const Buf& x = b == 0 ? h->emb : h->blk[b - 1].xout;
    prof_begin(c, "st_ln2_ff_bwd_b", b);
    {
      const bool last = b == h->nblk - 1;
      const float* dy[4] = {last ? nullptr : c.ws + h->dz1.off, last ? nullptr : c.ws + h->dxq.off, last ? nullptr : c.ws + h->dxk.off,
                            last ? nullptr : c.ws + h->dxv.off};
      DIB_CUDA_OK(ln_bwd(ln_args(c, k.hh, k.ff[nf], k.g2, k.be2, k.xout, k.mean2, k.rstd2), dy, last ? c.ws + h->d_pooled.off : nullptr,
                         h->dz2, &h->d_ff[nf], k.g2, k.be2));
    }
    if (stack_backward(c, k.ff_stack, sp)) return 1;
    prof_end(c);
    prof_begin(c, "st_ln1_out_proj_bwd_b", b);
    {
      const float* dy[4] = {c.ws + h->dz2.off, c.ws + h->dh_ff.off, nullptr, nullptr};
      DIB_CUDA_OK(ln_bwd(ln_args(c, x, k.a, k.g1, k.be1, k.hh, k.mean1, k.rstd1), dy, nullptr, h->dz1, nullptr, k.g1, k.be1));
    }
    if (stack_backward(c, k.o_stack, sp)) return 1;
    prof_end(c);
    prof_begin(c, "st_attn_bwd_b", b);
    DIB_CUDA_OK(h->varlen ? dib_launch_attn_varlen_bwd(attn_args(c, k), c.st) : dib_launch_attn_bwd(attn_args(c, k), c.st));
    prof_end(c);
    prof_begin(c, "st_qkv_bwd_b", b);
    if (stack_backward(c, k.qkv_stack, sp)) return 1;
    prof_end(c);
  }
  // d emb = block 0's residual-path gradient + its Q / K / V input gradients (dib_create requires at least one block)
  DibSumRows s;
  s.dst = c.ws + h->d_emb.off; s.count = (long long)c.n * h->d_emb.ld;
  s.src[0] = c.ws + h->dz1.off; s.src[1] = c.ws + h->dxq.off; s.src[2] = c.ws + h->dxk.off; s.src[3] = c.ws + h->dxv.off;
  prof_begin(c, "st_d_emb");
  DIB_CUDA_OK(dib_launch_sum_rows(s, c.st));
  prof_end(c);
  return 0;
}

// the forward of a call: the encoders (and a set transformer's attention blocks) on its particle rows, the integration network
// on its own rows
// forward_loss and, with compiled metrics and targets, the metric tail behind the stats row from the prediction the loss
// kernels wrote (into user_pred when the caller wants it, else into the workspace)
int forward_integration(const Ctx& c, const float* y, float inv_batch, bool training, float* user_pred, float* out_stats,
                        int nblk_kl) {
  dib_model* h = c.h;
  if (h->metrics.count == 0 || !y) return forward_loss(c, y, inv_batch, training, user_pred, out_stats, nblk_kl);
  float* z = user_pred ? user_pred : c.ws + h->metric_z_off;
  if (forward_loss(c, y, inv_batch, training, z, out_stats, nblk_kl)) return 1;
  prof_begin(c, "metrics");
  DIB_CUDA_OK(dib_launch_metrics(h->metrics, z, y, h->out, c.n, h->sample_weights_dev, c.ws + h->metric_part_off,
                                 h->d_metric_counter, out_stats + h->F + 3, c.st));
  prof_end(c);
  return 0;
}

int run_forward(const Ctx& c, const float* x, const float* y, const NoiseKey& nk, float inv_batch, float* user_pred,
                float* user_emb, float* out_stats, bool enc_only = false) {
  dib_model* h = c.h;
  const RowView r = particle_rows(c, nk);
  if (!h->route.int16 && tf32_shadow(c)) return 1;     // the 16-bit route runs no TF32 GEMM
  int nblk_kl = 0;
  if (forward_encoders(r.c, x, r.nk, user_emb, enc_only, &nblk_kl)) return 1;
  if (enc_only) {
    DIB_CUDA_OK(dib_launch_finalize_stats(c.ws + h->kl_part_off, h->kl_stride, nblk_kl, c.ws + h->loss_part_off,
                                          c.ws + h->acc_part_off, 0, h->F, c.n, 0, out_stats, c.st));
    return 0;
  }
  if (h->st && forward_set_blocks(r.c)) return 1;
  return forward_integration(c, y, inv_batch, nk.training, user_pred, out_stats, nblk_kl);
}

// the reverse mode of dib_train_step after its forward (and, with DIB_LOSS_INFONCE, the InfoNCE gradients) left the
// workspace: the IB weight from the stats, the integration network's, the output encoder's, the attention blocks' and the
// encoders' backward and the fixed-order reductions into grads_flat
int backward_all(const Ctx& c, const float* x, const NoiseKey& nk, const float* beta_dev, const float* stats, float inv_global_batch,
                 float* grads_flat) {
  dib_model* h = c.h;
  const RowView r = particle_rows(c, nk);
  const float* beta_w = nullptr;           // weight of the per-sample KL gradients in the encoder backward
  if (ib_weight(c, beta_dev, stats, inv_global_batch, &beta_w)) return 1;
  const Split sp = batch_split(c.n), sp_rows = batch_split(r.c.n);
  std::vector<DibReduceSeg> segs;          // fixed-order reductions of the step, run as ONE launch at the end
  if (backward_integration(c, inv_global_batch, sp, grads_flat, &segs)) return 1;
  if (infonce(h) && backward_output_encoder(c, sp, grads_flat)) return 1;
  if (h->st && backward_set_blocks(r.c, sp_rows)) return 1;
  int nrows = 0;
  const bool d16 = h->route.int16;         // the 16-bit integration backward leaves d emb in fp16
  if (backward_encoders(r.c, x, r.nk, d16 ? nullptr : c.ws + h->d_emb.off, d16 ? 0 : h->d_emb.ld, d16 ? c.ws + h->demb16_off : nullptr,
                        beta_w, inv_global_batch, sp_rows, &nrows))
    return 1;
  float* part = c.ws + h->part_off;
  const long long p_enc = h->intW[0];      // encoder (and attention block) parameters occupy [0, p_enc)
  prof_begin(c, "enc_split_reduce");
  if (h->route.enc_fused) {
    segs.push_back({part, h->Pp, nrows, p_enc, 1.f, grads_flat});
    DIB_CUDA_OK(dib_launch_reduce_segments(segs.data(), (int)segs.size(), c.st));
  } else {
    DIB_CUDA_OK(dib_launch_reduce_partials(part, h->Pp, nrows, p_enc, grads_flat, c.st));
  }
  prof_end(c);
  return 0;
}

// ---- DIB_LOSS_INFONCE across a data-parallel group (DESIGN section 7): the step split where rows of other ranks enter ----
int check_shard(const dib_model* h, const char* fn, int64_t n, int64_t n_global, int64_t row_offset, const void* e_all,
                const void* workspace) {
  if (!h) return fail("null model handle");
  if (!infonce(h)) return fail(std::string(fn) + ": the loss is not DIB_LOSS_INFONCE");
  if (n < 1 || n > h->maxB)
    return fail(std::string(fn) + ": n = " + std::to_string(n) + " must be in [1, config.max_batch = " + std::to_string(h->maxB) + "]");
  if (row_offset < 0 || n_global > 0x7fffffffll || row_offset + n > n_global)
    return fail(std::string(fn) + ": needs 0 <= row_offset and row_offset + n <= n_global < 2^31 (row_offset = " +
                std::to_string(row_offset) + ", n = " + std::to_string(n) + ", n_global = " + std::to_string(n_global) + ")");
  if (!e_all || (reinterpret_cast<uintptr_t>(e_all) & 15)) return fail(std::string(fn) + ": e_all must be 16-byte aligned");
  if (!workspace || (reinterpret_cast<uintptr_t>(workspace) & 255)) return fail(std::string(fn) + ": workspace must be 256-byte aligned");
  return 0;
}

// [e1 | e2] of all n_global rows, row-major [n_global, 2d]
DibInfonceStream shard_args(const Ctx& c, const float* e_all, int64_t n_global, int64_t row_offset, const float* lse_all) {
  const int d = c.h->out;
  float* lse = const_cast<float*>(lse_all);
  return infonce_args(c, e_all, 2 * d, e_all + d, 2 * d, n_global, row_offset, lse, lse + 1, 2);
}

}  // namespace

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

// =================================================================================================
void dib_note_launch(int n) { g_launches.fetch_add((unsigned long long)n, std::memory_order_relaxed); }

extern "C" {

uint64_t dib_launch_count(void) { return g_launches.load(); }

// bring-up switch (bit mask documented in include/dib_b200.h): this handle's reference kernels instead of the fused ones
int dib_debug_force_unfused(dib_model* h, int32_t on) {
  if (!h) return fail("null model handle");
  set_route(h, on);
  return 0;
}

int dib_profile_enable(dib_model* h, int32_t on) {
  if (!h) return fail("null model handle");
  for (auto& r : h->prof) { cudaEventDestroy(r.a); cudaEventDestroy(r.b); }
  h->prof.clear();
  h->profiling = on != 0;
  return 0;
}

int32_t dib_profile_read(dib_model* h, char* labels, size_t labels_bytes, float* ms, int32_t capacity) {
  if (!h) { fail("null model handle"); return -1; }
  std::string all;
  int32_t n = 0;
  for (auto& r : h->prof) {
    if (n >= capacity) break;
    if (cudaEventSynchronize(r.b) != cudaSuccess) { fail("dib_profile_read: event sync failed"); return -1; }
    float t = 0.f;
    cudaEventElapsedTime(&t, r.a, r.b);
    ms[n++] = t;
    all += r.label; all += '\n';
  }
  if (labels && labels_bytes) {
    const size_t k = all.size() < labels_bytes - 1 ? all.size() : labels_bytes - 1;
    memcpy(labels, all.data(), k); labels[k] = 0;
  }
  return n;
}

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
  if (kernel != DIB_GEMM_KERNEL_SIMT && kernel != DIB_GEMM_KERNEL_TC) return fail("dib_debug_gemm: unknown kernel");
  if (mode < DIB_GEMM_FWD || mode > DIB_GEMM_WGRAD) return fail("dib_debug_gemm: unknown mode");
  if (!problems || nprob < 1 || M < 0 || nsplit < 1) return fail("dib_debug_gemm: needs nprob >= 1, M >= 0 and nsplit >= 1");
  if (kernel == DIB_GEMM_KERNEL_SIMT && mode == DIB_GEMM_FWD && bias && bias != B)
    return fail("dib_debug_gemm: the simt kernel reads FWD biases from B's base (bias must be B or null)");
  const DibGemmProblem* hp = reinterpret_cast<const DibGemmProblem*>(problems);
  const cudaStream_t st = static_cast<cudaStream_t>(stream);
  if (kernel == DIB_GEMM_KERNEL_TC && !dib_gemm_tc_eligible(mode, hp, nprob, nullptr))
    return fail("dib_debug_gemm: the tensor-core kernel cannot run this group");
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
  cudaError_t e2 = cudaStreamSynchronize(st);
  cudaFree(dp);
  if (e != cudaSuccess) return fail(std::string("launch: ") + cudaGetErrorString(e));
  if (e2 != cudaSuccess) return fail(std::string("sync: ") + cudaGetErrorString(e2));
  return 0;
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
  const cudaError_t es = cudaStreamSynchronize(st);
  if (e != cudaSuccess) return fail(std::string("launch: ") + cudaGetErrorString(e));
  if (es != cudaSuccess) return fail(std::string("sync: ") + cudaGetErrorString(es));
  return 0;
}

// the attention core of a set-transformer block, fixed-size or key-tiled, through the launchers the steps use (unit tests)
int dib_debug_set_attention(int32_t variable_sizes, int32_t phases, const float* q, const float* k, const float* v,
                            const float* dout, int32_t ld, int64_t sets, int32_t heads, int32_t L, int32_t dk,
                            const int32_t* set_sizes, float* o, float* lse, float* dq, float* dk_, float* dv, float* dsum,
                            int32_t round_out, void* stream) {
  const std::string fn = "dib_debug_set_attention: ";
  if (variable_sizes != 0 && variable_sizes != 1) return fail(fn + "variable_sizes is 0 (fixed-size kernels) or 1 (key-tiled)");
  if (phases < 1 || phases > 3) return fail(fn + "phases is a mask of 1 (forward) and 2 (backward)");
  const int maxL = variable_sizes ? DIB_MAX_VARIABLE_SET_SIZE : 64;
  if (L < 1 || L > maxL) return fail(fn + "needs 1 <= L <= " + std::to_string(maxL) + " (L = " + std::to_string(L) + ")");
  if (dk < 1 || dk > 128) return fail(fn + "needs 1 <= dk <= 128 (dk = " + std::to_string(dk) + ")");
  if (heads < 1) return fail(fn + "needs heads >= 1");
  if ((heads * dk) % 4) return fail(fn + "needs heads * dk to be a multiple of 4 (heads * dk = " + std::to_string(heads * dk) + ")");
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
  const cudaError_t es = cudaStreamSynchronize(st);
  if (e != cudaSuccess) return fail(std::string("launch: ") + cudaGetErrorString(e));
  if (es != cudaSuccess) return fail(std::string("sync: ") + cudaGetErrorString(es));
  return 0;
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
  if (E < 1 || E > 128 || E % 4) return fail(fn + "needs 1 <= E <= 128, a multiple of 4 (E = " + std::to_string(E) + ")");
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
  const cudaError_t es = cudaStreamSynchronize(st);
  if (e != cudaSuccess) return fail(std::string("launch: ") + cudaGetErrorString(e));
  if (es != cudaSuccess) return fail(std::string("sync: ") + cudaGetErrorString(es));
  return 0;
}

// the mean over each set's rows (fixed or variable sizes) or zero_pad_rows, through the launchers the steps use (unit tests)
int dib_debug_set_pool(int32_t zero_pad, float* x, int32_t ld, int32_t E, int32_t L, int64_t sets, const int32_t* set_sizes,
                       float* out, int32_t ldo, int32_t round_out, void* stream) {
  const std::string fn = "dib_debug_set_pool: ";
  const int maxL = set_sizes ? DIB_MAX_VARIABLE_SET_SIZE : 64;
  if (zero_pad != 0 && zero_pad != 1) return fail(fn + "zero_pad is 0 (mean pooling) or 1 (zero_pad_rows)");
  if (zero_pad && !set_sizes) return fail(fn + "zero_pad_rows needs set_sizes");
  if (L < 1 || L > maxL) return fail(fn + "needs 1 <= L <= " + std::to_string(maxL) + " (L = " + std::to_string(L) + ")");
  if (sets < 0 || sets > 65535) return fail(fn + "needs 0 <= sets <= 65535 (sets = " + std::to_string(sets) + ")");
  if (!x) return fail(fn + "x must not be null");
  if (!zero_pad && (E < 1 || E > 128 || E % 4 || ld < E || ldo < E || !out))
    return fail(fn + "mean pooling needs 1 <= E <= 128 a multiple of 4, ld >= E, ldo >= E and out");
  if (zero_pad && ld < 1) return fail(fn + "needs ld >= 1");
  const cudaStream_t st = static_cast<cudaStream_t>(stream);
  cudaError_t e;
  if (zero_pad) e = dib_launch_zero_pad_rows(x, ld, sets * L, L, set_sizes, st);
  else if (set_sizes) e = dib_launch_pool_varlen_fwd(x, ld, E, L, sets, set_sizes, out, ldo, round_out ? 1 : 0, st);
  else e = dib_launch_pool_fwd(x, ld, E, L, sets, out, ldo, round_out ? 1 : 0, st);
  const cudaError_t es = cudaStreamSynchronize(st);
  if (e != cudaSuccess) return fail(std::string("launch: ") + cudaGetErrorString(e));
  if (es != cudaSuccess) return fail(std::string("sync: ") + cudaGetErrorString(es));
  return 0;
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
  const cudaError_t es = cudaStreamSynchronize(st);
  if (e != cudaSuccess) return fail(std::string("launch: ") + cudaGetErrorString(e));
  if (es != cudaSuccess) return fail(std::string("sync: ") + cudaGetErrorString(es));
  return 0;
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
  const cudaError_t es = cudaStreamSynchronize(st);
  if (e != cudaSuccess) return fail(std::string("launch: ") + cudaGetErrorString(e));
  if (es != cudaSuccess) return fail(std::string("sync: ") + cudaGetErrorString(es));
  return 0;
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
  const cudaError_t es = cudaStreamSynchronize(st);
  if (e != cudaSuccess) return fail(std::string("launch: ") + cudaGetErrorString(e));
  if (es != cudaSuccess) return fail(std::string("sync: ") + cudaGetErrorString(es));
  return 0;
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
  const cudaError_t es = cudaStreamSynchronize(st);
  if (e != cudaSuccess) return fail(std::string("launch: ") + cudaGetErrorString(e));
  if (es != cudaSuccess) return fail(std::string("sync: ") + cudaGetErrorString(es));
  return 0;
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
  const cudaError_t es = cudaStreamSynchronize(st);
  if (e != cudaSuccess) return fail(std::string("launch: ") + cudaGetErrorString(e));
  if (es != cudaSuccess) return fail(std::string("sync: ") + cudaGetErrorString(es));
  return 0;
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


#define DIB_HOOK_CHECK(msg)                          \
  do {                                               \
    const std::string _m = (msg);                    \
    if (!_m.empty()) return fail(fn + _m);           \
  } while (0)

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
      if (l.K < 64 || l.K % 64) return fail(fn + lq + "needs K a positive multiple of 64 (K = " + std::to_string(l.K) + ")");
      if (l.N < 128 || l.N % 128) return fail(fn + lq + "needs N a positive multiple of 128 (N = " + std::to_string(l.N) + ")");
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
  if (K < 64 || K % 64) return fail(fn + "needs K a positive multiple of 64 (K = " + std::to_string(K) + ")");
  if (N < 128 || N % 128) return fail(fn + "needs N a positive multiple of 128 (N = " + std::to_string(N) + ")");
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
  if (K != 256) return fail(fn + "needs K == 256 (K = " + std::to_string(K) + ")");
  if (out_dim < 1 || out_dim > 16) return fail(fn + "needs 1 <= out_dim <= 16 (out_dim = " + std::to_string(out_dim) + ")");
  if (head1 && out_dim != 1) return fail(fn + "head1 needs out_dim == 1");
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
#undef DIB_HOOK_CHECK

const char* dib_last_error(void) { return g_last_error.c_str(); }

const char* dib_build_info(void) {
  return "dib_b200 abi=5 arch=sm_90a paths=fp32-simt,tf32-wgmma,fp16-fused-wgmma,bf16-fused-wgmma";
}

int32_t dib_model_info(const dib_model* h, char* out, size_t out_bytes) {
  if (!h || !out || out_bytes < 2) { fail("dib_model_info: bad arguments"); return -1; }
  static const char* pn[] = {"fp32", "tf32", "bf16", "fp16"};
  const bool fused = h->route.enc_fused, i16 = h->route.int16;
  const char* k16 = h->precision == DIB_PREC_BF16 ? "bf16" : "f16";
  std::string s = std::string("precision=") + pn[h->precision];
  if (!is_tc(h)) s += " encoders=simt-fp32 integration=simt-fp32 operands=fp32 accumulate=fp32";
  else {
    s += fused ? std::string(" encoders=fused-wgmma-") + k16 : std::string(" encoders=grouped-wgmma-tf32");
    s += i16 ? std::string(" integration=int16-wgmma-") + k16 : std::string(" integration=wgmma-tf32");
    s += fused ? std::string(" operands=") + (h->precision == DIB_PREC_BF16 ? "bf16" : "fp16") : std::string(" operands=tf32");
    s += " accumulate=fp32";
  }
  if (h->route.tail_fused) s += h->route.tail_bwd ? " integration_tail=fwd2-head-dgrad" : " integration_tail=fwd2-head";
  else if (h->route.int16) s += h->route.head1 ? " integration_head=head1" : " integration_head=generic";
  if (h->st)
    s += std::string(" set_transformer=") + (h->varlen ? "attention-varlen-simt-fp32" : "attention-simt-fp32") +
         ",layernorm-simt-fp32,dense-" + (is_tc(h) ? "wgmma-tf32" : "simt-fp32");
  if (infonce(h))
    s += std::string(" output_encoder=") + (is_tc(h) ? "wgmma-tf32" : "simt-fp32") + " loss=infonce-stream-fp32";
  const size_t k = s.size() < out_bytes - 1 ? s.size() : out_bytes - 1;
  memcpy(out, s.data(), k); out[k] = 0;
  return (int32_t)k;
}

int dib_create(const dib_config* cfg, dib_model** out) {
  if (!cfg || !out) return fail("dib_create: null argument");
  *out = nullptr;
  // an abi_version 2 struct ends before the InfoNCE fields: read only its prefix
  if (cfg->abi_version < 2 || cfg->abi_version > DIB_ABI_VERSION) return fail("dib_create: abi_version mismatch");
  const int kind = cfg->abi_version >= 4 ? cfg->integration_kind : DIB_INTEGRATION_MLP;
  if (kind != DIB_INTEGRATION_MLP && kind != DIB_INTEGRATION_SET_TRANSFORMER) return fail("dib_create: unknown integration_kind");
  const bool varlen = cfg->abi_version >= 5 && cfg->variable_set_sizes != 0;
  if (varlen && kind != DIB_INTEGRATION_SET_TRANSFORMER) return fail("dib_create: variable_set_sizes needs the set transformer");
  if (kind == DIB_INTEGRATION_SET_TRANSFORMER) {
    const int E = cfg->feature_embedding_dimension;
    if (varlen && (cfg->set_size < 1 || cfg->set_size > DIB_MAX_VARIABLE_SET_SIZE))
      return fail("dib_create: set transformer with variable set sizes needs set_size (the largest set) in [1, " +
                  std::to_string(DIB_MAX_VARIABLE_SET_SIZE) + "]");
    if (!varlen && (cfg->set_size < 1 || cfg->set_size > 64))
      return fail("dib_create: set transformer needs set_size in [1, 64] (up to " + std::to_string(DIB_MAX_VARIABLE_SET_SIZE) +
                  " with variable_set_sizes)");
    if (cfg->number_features != 1) return fail("dib_create: set transformer needs number_features == 1 (one shared particle encoder)");
    if (cfg->number_attention_blocks < 1 || cfg->number_heads < 1 || cfg->key_dim < 1 || cfg->key_dim > 128)
      return fail("dib_create: set transformer needs >= 1 attention block, >= 1 head and key_dim in [1, 128]");
    if (((long long)cfg->number_heads * cfg->key_dim) % 4 || E % 4 || E > 128)
      return fail("dib_create: set transformer needs number_heads * key_dim and E multiples of 4 and E <= 128");
    if (cfg->number_ff_layers < 1 || !cfg->ff_architecture || cfg->ff_architecture[cfg->number_ff_layers - 1] != E)
      return fail("dib_create: set transformer needs an FF stack whose last width equals E (the residual adds it to the input)");
    for (int j = 0; j < cfg->number_ff_layers; ++j)
      if (cfg->ff_architecture[j] < 1) return fail("dib_create: FF width < 1");
    if (cfg->ff_activation_fn < 0 || cfg->ff_activation_fn > DIB_ACT_ELU) return fail("dib_create: unknown FF activation");
    if (cfg->loss == DIB_LOSS_SPARSE_CE_LOGITS || cfg->loss == DIB_LOSS_INFONCE)
      return fail("dib_create: set transformer supports BCE (logits or probabilities), MSE and the external loss");
    if (cfg->dropout_rate != 0.f) return fail("dib_create: set transformer has no dropout");
    if (cfg->max_batch > 65535 || cfg->max_batch * cfg->set_size > 0x7fffffffll)
      return fail("dib_create: set transformer needs max_batch <= 65535 sets");
    if (!(cfg->layer_norm_epsilon >= 0.f)) return fail("dib_create: layer_norm_epsilon must be >= 0");
  }
  if (cfg->number_features < 1 || cfg->feature_embedding_dimension < 1 || cfg->output_dimensionality < 1 ||
      cfg->max_batch < 1 || cfg->number_encoder_layers < 0 || cfg->number_integration_layers < 0)
    return fail("dib_create: invalid sizes");
  if (cfg->max_batch > 0x7fffffffll) return fail("dib_create: max_batch too large");
  // the reparametrisation and KL kernels index the feature by gridDim.y, whose hardware limit is 65 535
  if (cfg->number_features > 65535)
    return fail("dib_create: number_features = " + std::to_string(cfg->number_features) + " exceeds 65535");
  if (cfg->precision < DIB_PREC_FP32 || cfg->precision > DIB_PREC_FP16)
    return fail("dib_create: unknown precision");
  if (cfg->activation_fn < 0 || cfg->activation_fn > DIB_ACT_ELU || cfg->output_activation_fn < 0 ||
      cfg->output_activation_fn > DIB_ACT_ELU)
    return fail("dib_create: unknown activation");
  if (cfg->loss < 0 || cfg->loss > DIB_LOSS_INFONCE || (cfg->loss == DIB_LOSS_INFONCE && cfg->abi_version < 3))
    return fail("dib_create: unknown loss");
  if (cfg->loss == DIB_LOSS_INFONCE) {
    if (cfg->y_dimensionality < 1 || cfg->number_y_encoder_layers < 0 || (cfg->number_y_encoder_layers > 0 && !cfg->y_encoder_architecture))
      return fail("dib_create: InfoNCE needs y_dimensionality >= 1 and an output-encoder architecture");
    for (int j = 0; j < cfg->number_y_encoder_layers; ++j)
      if (cfg->y_encoder_architecture[j] < 1) return fail("dib_create: output-encoder width < 1");
    if (cfg->infonce_similarity < 0 || cfg->infonce_similarity > 4) return fail("dib_create: unknown InfoNCE similarity");
    if (!(cfg->infonce_temperature > 0.f)) return fail("dib_create: InfoNCE temperature must be > 0");
    if (cfg->output_dimensionality > 512) return fail("dib_create: InfoNCE needs output_dimensionality <= 512");
    if (cfg->output_activation_fn != DIB_ACT_LINEAR) return fail("dib_create: InfoNCE needs a linear output (train.py:117)");
  }
  dib_model* h = new (std::nothrow) dib_model();
  if (!h) return fail("dib_create: out of host memory");
  h->F = cfg->number_features; h->L = cfg->number_encoder_layers; h->Li = cfg->number_integration_layers;
  h->E = cfg->feature_embedding_dimension; h->out = cfg->output_dimensionality;
  h->act = cfg->activation_fn; h->out_act = cfg->output_activation_fn; h->loss = cfg->loss;
  h->precision = cfg->precision; h->use_pe = cfg->use_positional_encoding ? 1 : 0;
  h->alpha = cfg->leaky_relu_alpha; h->maxB = cfg->max_batch;
  h->lv_off = cfg->logvar_offset;
  h->kl_exp = cfg->kl_loss_exponent == 0.f ? 1.f : cfg->kl_loss_exponent;
  h->kl_scale = cfg->kl_loss_scale == 0.f ? 1.f : cfg->kl_loss_scale;
  h->simple = cfg->encoder_kind == DIB_ENCODER_SIMPLE;
  h->drop = cfg->dropout_rate;
  if (infonce(h)) {
    h->ydim = cfg->y_dimensionality; h->Ly = cfg->number_y_encoder_layers;
    h->y_arch.assign(cfg->y_encoder_architecture, cfg->y_encoder_architecture + h->Ly);
    h->sim_kind = cfg->infonce_similarity; h->temperature = cfg->infonce_temperature;
  }
  if (kind == DIB_INTEGRATION_SET_TRANSFORMER) {
    h->st = true;
    h->varlen = varlen;
    h->Ls = cfg->set_size; h->nblk = cfg->number_attention_blocks; h->heads = cfg->number_heads; h->dkey = cfg->key_dim;
    h->hdk = h->heads * h->dkey;
    h->ff_arch.assign(cfg->ff_architecture, cfg->ff_architecture + cfg->number_ff_layers);
    h->ff_act = cfg->ff_activation_fn;
    h->ln_eps = cfg->layer_norm_epsilon == 0.f ? 1e-3f : cfg->layer_norm_epsilon;
    h->maxSets = cfg->max_batch;
    h->maxB = cfg->max_batch * h->Ls;      // encoder and block buffers hold particle rows
    h->blk.assign(h->nblk, dib_model::StBlock());
  }
  if (!(h->drop >= 0.f && h->drop < 1.f)) { delete h; return fail("dib_create: dropout_rate must be in [0, 1)"); }
  if (cfg->encoder_kind != DIB_ENCODER_MLP && cfg->encoder_kind != DIB_ENCODER_SIMPLE) { delete h; return fail("dib_create: unknown encoder_kind"); }
  if (!(h->kl_exp > 0.f)) { delete h; return fail("dib_create: kl_loss_exponent must be > 0"); }
  if (h->simple) { h->L = 0; h->use_pe = 0; }
  // models.py:70: frequencies 2**arange(1, n) -> n-1 sinusoid blocks after the identity block
  h->nfreq = h->use_pe ? (cfg->number_positional_encoding_frequencies > 1 ? cfg->number_positional_encoding_frequencies : 1) : 1;
  h->fdims.assign(cfg->feature_dimensionalities, cfg->feature_dimensionalities + h->F);
  h->enc_arch.assign(cfg->feature_encoder_architecture, cfg->feature_encoder_architecture + h->L);
  if (h->simple) for (int d : h->fdims) if (d != h->E) { delete h; return fail("dib_create: SimpleEncoder needs d_i == feature_embedding_dimension"); }
  h->int_arch.assign(cfg->integration_network_architecture, cfg->integration_network_architecture + h->Li);
  for (int d : h->fdims) if (d < 1) { delete h; return fail("dib_create: feature dimensionality < 1"); }
  for (int d : h->enc_arch) if (d < 1) { delete h; return fail("dib_create: encoder width < 1"); }
  for (int d : h->int_arch) if (d < 1) { delete h; return fail("dib_create: integration width < 1"); }

  // first-layer operand layout: per feature a zero-padded block of width round_up(d_i * nfreq, 4)
  std::vector<int> col_src, col_freq, col_feat;
  h->D = 0;
  for (int f = 0; f < h->F; ++f) {
    const int d = h->fdims[f], w = d * h->nfreq;
    h->x_off.push_back(h->D);
    h->pe_off.push_back((int)col_src.size());
    h->w_in.push_back(w);
    for (int blk = 0; blk < h->nfreq; ++blk)
      for (int k = 0; k < d; ++k) { col_src.push_back(h->D + k); col_freq.push_back(blk == 0 ? 0 : (1 << blk)); }
    while (col_src.size() % 4) { col_src.push_back(-1); col_freq.push_back(0); }
    col_feat.resize(col_src.size(), f);
    h->D += d;
  }
  h->ldpe = (int)col_src.size();
  // the output encoder's positional encoding: one block per frequency over the y columns (train.py:187-188)
  std::vector<int> ycol_src, ycol_freq;
  for (int blk = 0; infonce(h) && blk < h->nfreq; ++blk)
    for (int k = 0; k < h->ydim; ++k) { ycol_src.push_back(k); ycol_freq.push_back(blk == 0 ? 0 : (1 << blk)); }
  while (ycol_src.size() % 4) { ycol_src.push_back(-1); ycol_freq.push_back(0); }
  h->ldype = (int)ycol_src.size();

  // flat parameter layout (Keras variable order: per feature W,b per layer; then the integration network)
  long long off = 0;
  auto add_var = [&](int rows, int cols) {
    h->var_off.push_back(off); h->var_rows.push_back(rows); h->var_cols.push_back(cols);
    const long long o = off; off += (long long)(rows ? rows : 1) * cols; return o;
  };
  h->encW.assign(h->F, {}); h->encB.assign(h->F, {});
  for (int f = 0; f < h->F; ++f) {
    if (h->simple) {                       // nb-bool cell 4: mu_scaling (1,1), logvar (1,1)
      h->encW[f].push_back(add_var(1, 1));
      h->encB[f].push_back(add_var(1, 1));
      continue;
    }
    for (int j = 0; j <= h->L; ++j) {
      h->encW[f].push_back(add_var(enc_fan_in(h, f, j), enc_fan_out(h, j)));
      h->encB[f].push_back(add_var(0, enc_fan_out(h, j)));
    }
  }
  for (auto& k : h->blk) {                 // Keras functional order inside each attention block
    k.Wq = add_var(h->E, h->hdk); k.bq = add_var(0, h->hdk);
    k.Wk = add_var(h->E, h->hdk); k.bk = add_var(0, h->hdk);
    k.Wv = add_var(h->E, h->hdk); k.bv = add_var(0, h->hdk);
    k.Wo = add_var(h->hdk, h->E); k.bo = add_var(0, h->E);
    k.g1 = add_var(0, h->E); k.be1 = add_var(0, h->E);
    for (int j = 0; j < nff(h); ++j) { k.ffW.push_back(add_var(ff_fan_in(h, j), h->ff_arch[j])); k.ffB.push_back(add_var(0, h->ff_arch[j])); }
    k.g2 = add_var(0, h->E); k.be2 = add_var(0, h->E);
  }
  for (int j = 0; j <= h->Li; ++j) {
    h->intW.push_back(add_var(int_fan_in(h, j), int_fan_out(h, j)));
    h->intB.push_back(add_var(0, int_fan_out(h, j)));
  }
  h->Px = off;
  for (int j = 0; infonce(h) && j <= h->Ly; ++j) {     // all_trainable_variables = model + output_encoder (train.py:198)
    h->yW.push_back(add_var(y_fan_in(h, j), y_fan_out(h, j)));
    h->yB.push_back(add_var(0, y_fan_out(h, j)));
  }
  h->P = off; h->Pp = DIB_ROUND_UP(off, 64);
  {
    int dev = 0;
    cudaGetDevice(&dev);
    if (cudaDeviceGetAttribute(&h->num_sms, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || h->num_sms < 1)
      h->num_sms = 132;
  }
  plan(h);

  std::vector<DibGemmProblem> probs;
  build_problems(h, probs);
  h->h_probs = probs;
  cudaError_t e = cudaMalloc(&h->d_probs, probs.size() * sizeof(DibGemmProblem));
  if (e == cudaSuccess) e = cudaMalloc(&h->d_col_src, col_src.size() * sizeof(int));
  if (e == cudaSuccess) e = cudaMalloc(&h->d_col_freq, col_freq.size() * sizeof(int));
  if (e == cudaSuccess) e = cudaMalloc(&h->d_col_feat, col_feat.size() * sizeof(int));
  if (e == cudaSuccess) e = cudaMalloc(&h->d_xoff, h->x_off.size() * sizeof(int));
  if (e == cudaSuccess) e = cudaMemcpy(h->d_xoff, h->x_off.data(), h->x_off.size() * sizeof(int), cudaMemcpyHostToDevice);
  if (e == cudaSuccess) e = cudaMemcpy(h->d_probs, probs.data(), probs.size() * sizeof(DibGemmProblem), cudaMemcpyHostToDevice);
  if (e == cudaSuccess) e = cudaMemcpy(h->d_col_src, col_src.data(), col_src.size() * sizeof(int), cudaMemcpyHostToDevice);
  if (e == cudaSuccess) e = cudaMemcpy(h->d_col_freq, col_freq.data(), col_freq.size() * sizeof(int), cudaMemcpyHostToDevice);
  if (e == cudaSuccess) e = cudaMemcpy(h->d_col_feat, col_feat.data(), col_feat.size() * sizeof(int), cudaMemcpyHostToDevice);
  if (e == cudaSuccess && infonce(h)) {
    e = cudaMalloc(&h->d_ycol_src, ycol_src.size() * sizeof(int));
    if (e == cudaSuccess) e = cudaMalloc(&h->d_ycol_freq, ycol_freq.size() * sizeof(int));
    if (e == cudaSuccess) e = cudaMemcpy(h->d_ycol_src, ycol_src.data(), ycol_src.size() * sizeof(int), cudaMemcpyHostToDevice);
    if (e == cudaSuccess) e = cudaMemcpy(h->d_ycol_freq, ycol_freq.data(), ycol_freq.size() * sizeof(int), cudaMemcpyHostToDevice);
  }
  if (e == cudaSuccess && h->st) e = h->varlen ? dib_attn_varlen_prepare() : dib_attn_prepare();
  if (e != cudaSuccess) {
    std::string msg = std::string("dib_create: CUDA error: ") + cudaGetErrorString(e);
    dib_destroy(h);
    return fail(msg);
  }
  // ---- fused encoder kernels: two hidden layers of 128, E = 32, first-layer fan-in (+ bias column) <= 16
  {
    bool ok = want16(h) && !h->st && h->drop == 0.f && h->L == 2 && h->enc_arch[0] == 128 && h->enc_arch[1] == 128 && h->E == 32;
    for (int f = 0; ok && f < h->F; ++f) ok = h->w_in[f] + 1 <= 16;
    if (ok) {
      const int F = h->F;
      std::vector<long long> tab(6 * (size_t)F);
      std::vector<int> itab(2 * (size_t)F);
      for (int f = 0; f < F; ++f) {
        tab[0 * F + f] = h->encW[f][0]; tab[1 * F + f] = h->encB[f][0]; tab[2 * F + f] = h->encW[f][1];
        tab[3 * F + f] = h->encB[f][1]; tab[4 * F + f] = h->encW[f][2]; tab[5 * F + f] = h->encB[f][2];
        itab[f] = h->x_off[f]; itab[F + f] = h->fdims[f];
      }
      const size_t b1 = tab.size() * sizeof(long long), b2 = itab.size() * sizeof(int);
      cudaError_t fe = cudaMalloc(&h->d_fused_tables, b1 + b2);
      if (fe == cudaSuccess) fe = cudaMemcpy(h->d_fused_tables, tab.data(), b1, cudaMemcpyHostToDevice);
      if (fe == cudaSuccess) fe = cudaMemcpy(static_cast<char*>(h->d_fused_tables) + b1, itab.data(), b2, cudaMemcpyHostToDevice);
      if (fe == cudaSuccess) {
        const long long* lt = static_cast<const long long*>(h->d_fused_tables);
        const int* it = reinterpret_cast<const int*>(static_cast<const char*>(h->d_fused_tables) + b1);
        DibEncFusedDesc& d = h->fdesc;
        d.F = F; d.nfreq = h->nfreq; d.act = h->act; d.alpha = h->alpha; d.bf16 = h->precision == DIB_PREC_BF16 ? 1 : 0;
        d.w0_off = lt; d.b0_off = lt + F; d.w1_off = lt + 2 * F; d.b1_off = lt + 3 * F; d.w2_off = lt + 4 * F;
        d.b2_off = lt + 5 * F; d.x_off = it; d.fdim = it + F;
        h->fused_ok = true;
        // 16-bit integration path: hidden widths multiples of 128, last hidden width 256, narrow output head
        // (the fused head owns the compiled loss, so a caller-owned loss and InfoNCE take the TF32 integration kernels)
        bool iok = h->Li >= 1 && (h->F * h->E) % 64 == 0 && h->int_arch[h->Li - 1] == 256 && h->out <= 16 &&
                   h->loss != DIB_LOSS_EXTERNAL && h->loss != DIB_LOSS_INFONCE;
        for (int j = 0; iok && j < h->Li; ++j) iok = h->int_arch[j] % 128 == 0 && (h->intB[j] & 3) == 0;
        h->int16_ok = iok;
      }
    }
  }
  set_route(h, 0);
  *out = h;
  return 0;
}

void dib_destroy(dib_model* h) {
  if (!h) return;
  if (h->d_probs) cudaFree(h->d_probs);
  if (h->d_col_src) cudaFree(h->d_col_src);
  if (h->d_col_freq) cudaFree(h->d_col_freq);
  if (h->d_col_feat) cudaFree(h->d_col_feat);
  if (h->d_xoff) cudaFree(h->d_xoff);
  if (h->d_fused_tables) cudaFree(h->d_fused_tables);
  if (h->d_ycol_src) cudaFree(h->d_ycol_src);
  if (h->d_ycol_freq) cudaFree(h->d_ycol_freq);
  if (h->d_metric_counter) cudaFree(h->d_metric_counter);
  for (auto& r : h->prof) { cudaEventDestroy(r.a); cudaEventDestroy(r.b); }
  delete h;
}

int64_t dib_param_count(const dib_model* h) { return h ? h->P : -1; }

int dib_param_layout(const dib_model* h, int64_t* offsets, int32_t* rows, int32_t* cols, int32_t capacity) {
  if (!h) { fail("null model handle"); return -1; }
  const int nv = (int)h->var_off.size();
  if (!offsets || !rows || !cols) return nv;
  if (capacity < nv) { fail("dib_param_layout: capacity too small"); return -1; }
  for (int i = 0; i < nv; ++i) { offsets[i] = h->var_off[i]; rows[i] = h->var_rows[i]; cols[i] = h->var_cols[i]; }
  return nv;
}

size_t dib_workspace_bytes(const dib_model* h) { return h ? (size_t)h->ws_floats * sizeof(float) : 0; }

int32_t dib_stats_count(const dib_model* h) { return h ? stats_count(h) : -1; }

int dib_forward(dib_model* h, const float* params, const float* x, const float* y, int64_t n, const float* beta_dev,
                const float* eps, uint64_t seed, uint32_t step, uint64_t sample_offset, float* out_pred, float* out_emb,
                float* out_stats, void* workspace, void* stream) {
  (void)beta_dev;
  if (check_call(h, params, x, n, workspace) || check_sets(h, n)) return 1;
  if (!out_stats) return fail("dib_forward: out_stats is required");
  Ctx c{h, params, static_cast<float*>(workspace), static_cast<cudaStream_t>(stream), (int)n};
  if (n == 0) { DIB_CUDA_OK(cudaMemsetAsync(out_stats, 0, sizeof(float) * stats_count(h), c.st)); return 0; }
  return run_forward(c, x, y, NoiseKey{eps, seed, step, sample_offset, false}, 0.f, out_pred, out_emb, out_stats);
}

int dib_encode_feature(dib_model* h, const float* params, int32_t feature, const float* x_i, int64_t n,
                       float* out_mu_logvar, void* workspace, void* stream) {
  if (check_call(h, params, x_i, n, workspace)) return 1;
  if (feature < 0 || feature >= h->F) return fail("dib_encode_feature: feature index out of range");
  if (!out_mu_logvar) return fail("dib_encode_feature: null output");
  if (n == 0) return 0;
  Ctx c{h, params, static_cast<float*>(workspace), static_cast<cudaStream_t>(stream), (int)n};
  const int f = feature;
  if (!h->simple && tf32_shadow(c)) return 1;
  if (encode_all(c, x_i, h->fdims[f], f, nullptr, 0)) return 1;
  DIB_CUDA_OK(dib_launch_copy2d(c.ws + h->enc_out.off + f * h->enc_out.feat_stride, h->enc_out.ld, out_mu_logvar,
                                2 * h->E, 2 * h->E, n, c.st));
  return 0;
}

int dib_train_step(dib_model* h, const float* params, const float* x, const float* y, int64_t n, const float* beta_dev,
                   float inv_global_batch, const float* eps, uint64_t seed, uint32_t step, uint64_t sample_offset,
                   float* grads_flat, float* out_stats, void* workspace, void* stream) {
  if (check_call(h, params, x, n, workspace) || check_sets(h, n)) return 1;
  if ((!y && n > 0) || !beta_dev || !grads_flat || !out_stats)
    return fail("dib_train_step: y, beta_dev, grads_flat and out_stats are required");
  Ctx c{h, params, static_cast<float*>(workspace), static_cast<cudaStream_t>(stream), (int)n};
  c.dev_step = true;
  if (n == 0) {
    DIB_CUDA_OK(cudaMemsetAsync(grads_flat, 0, sizeof(float) * h->P, c.st));
    DIB_CUDA_OK(cudaMemsetAsync(out_stats, 0, sizeof(float) * stats_count(h), c.st));
    return 0;
  }
  const NoiseKey nk{eps, seed, step, sample_offset, true};
  if (run_forward(c, x, y, nk, inv_global_batch, nullptr, nullptr, out_stats)) return 1;
  return backward_all(c, x, nk, beta_dev, out_stats, inv_global_batch, grads_flat);
}

int dib_infonce_shard_forward(dib_model* h, const float* params, const float* x, const float* y, int64_t n, int32_t training,
                              const float* eps, uint64_t seed, uint32_t step, uint64_t sample_offset, float* e_all,
                              int64_t n_global, int64_t row_offset, void* workspace, void* stream) {
  if (check_call(h, params, x, n, workspace) ||
      check_shard(h, "dib_infonce_shard_forward", n, n_global, row_offset, e_all, workspace))
    return 1;
  if (!y) return fail("dib_infonce_shard_forward: y is required");
  Ctx c{h, params, static_cast<float*>(workspace), static_cast<cudaStream_t>(stream), (int)n};
  c.dev_step = training != 0;
  const NoiseKey nk{eps, seed, step, sample_offset, training != 0};
  if (!h->route.int16 && tf32_shadow(c)) return 1;
  int nblk_kl = 0;
  if (forward_encoders(c, x, nk, nullptr, false, &nblk_kl) || stack_forward(c, h->int_stack, 0, 1) || forward_output_encoder(c, y))
    return 1;
  h->nce_nblk_kl = nblk_kl;
  const int d = h->out;
  float* own = e_all + row_offset * 2 * d;
  DIB_CUDA_OK(dib_launch_copy2d(c.ws + h->pred.off, h->pred.ld, own, 2 * d, d, n, c.st));
  DIB_CUDA_OK(dib_launch_copy2d(c.ws + h->y_out.off, h->y_out.ld, own + d, 2 * d, d, n, c.st));
  return 0;
}

int dib_infonce_shard_lse(dib_model* h, const float* e_all, int64_t n_global, int64_t row_offset, int64_t n, float* lse_all,
                          float* out_stats, void* workspace, void* stream) {
  if (check_shard(h, "dib_infonce_shard_lse", n, n_global, row_offset, e_all, workspace)) return 1;
  if (!lse_all || (reinterpret_cast<uintptr_t>(lse_all) & 15) || !out_stats)
    return fail("dib_infonce_shard_lse: lse_all (16-byte aligned) and out_stats are required");
  Ctx c{h, nullptr, static_cast<float*>(workspace), static_cast<cudaStream_t>(stream), (int)n};
  if (infonce_loss_stats(c, shard_args(c, e_all, n_global, row_offset, lse_all), out_stats, h->nce_nblk_kl)) return 1;
  if (h->kl_exp != 1.f || h->kl_scale != 1.f)      // the backward's IB weight reads the KL sums
    DIB_CUDA_OK(cudaMemcpyAsync(c.ws + h->nce_stats_off, out_stats, sizeof(float) * (h->F + 3), cudaMemcpyDeviceToDevice, c.st));
  return 0;
}

int dib_infonce_shard_backward(dib_model* h, const float* params, const float* x, int64_t n, const float* beta_dev, const float* eps,
                               uint64_t seed, uint32_t step, uint64_t sample_offset, const float* e_all, const float* lse_all,
                               int64_t n_global, int64_t row_offset, float* grads_flat, void* workspace, void* stream) {
  if (check_call(h, params, x, n, workspace) ||
      check_shard(h, "dib_infonce_shard_backward", n, n_global, row_offset, e_all, workspace))
    return 1;
  if (!lse_all || (reinterpret_cast<uintptr_t>(lse_all) & 15) || !beta_dev || !grads_flat)
    return fail("dib_infonce_shard_backward: lse_all (16-byte aligned), beta_dev and grads_flat are required");
  Ctx c{h, params, static_cast<float*>(workspace), static_cast<cudaStream_t>(stream), (int)n};
  c.dev_step = true;
  const NoiseKey nk{eps, seed, step, sample_offset, true};
  if (infonce_grads(c, shard_args(c, e_all, n_global, row_offset, lse_all))) return 1;
  // rounded from double like a caller's inv_global_batch: one rank's step is dib_train_step's bit for bit
  return backward_all(c, x, nk, beta_dev, c.ws + h->nce_stats_off, (float)(1.0 / (double)n_global), grads_flat);
}

// Philox 'step' word from device memory (CUDA-Graph replay: a captured launch cannot carry a fresh by-value step):
// when set, every forward / train-step call uses step + *step_dev.  The caller owns and advances the counter.
int dib_set_noise_step_device(dib_model* h, const uint32_t* step_dev) {
  if (!h) return fail("null model handle");
  h->step_dev = step_dev;
  return 0;
}

// the int32 sizes of the n sets of the following calls, read by the kernels from device memory: a captured graph reads
// whatever the buffer holds at replay
int dib_set_set_sizes_device(dib_model* h, const int32_t* set_sizes_dev) {
  if (!h) return fail("null model handle");
  if (!h->varlen && set_sizes_dev) return fail("dib_set_set_sizes_device: the model was not created with variable_set_sizes");
  if (reinterpret_cast<uintptr_t>(set_sizes_dev) & 3) return fail("dib_set_set_sizes_device: sizes must be 4-byte aligned");
  h->set_sizes_dev = set_sizes_dev;
  return 0;
}

// the fp32 sample weights of the n rows of the following dib_forward / dib_train_step calls, read by the loss kernels from
// device memory (a captured graph reads whatever the buffer holds at replay); null: unweighted
int dib_set_sample_weights_device(dib_model* h, const float* w_dev) {
  if (!h) return fail("null model handle");
  if (w_dev && (h->loss == DIB_LOSS_EXTERNAL || h->loss == DIB_LOSS_INFONCE))
    return fail("dib_set_sample_weights_device: the external and InfoNCE losses take no sample weights");
  if (reinterpret_cast<uintptr_t>(w_dev) & 3) return fail("dib_set_sample_weights_device: weights must be 4-byte aligned");
  h->sample_weights_dev = w_dev;
  return 0;
}

int dib_set_metrics(dib_model* h, const dib_metric_spec* specs, int32_t count) {
  if (!h) return fail("null model handle");
  if (count < 0 || count > DIB_MAX_METRICS || (count > 0 && !specs))
    return fail("dib_set_metrics: 0 <= count <= DIB_MAX_METRICS specs are required");
  if (count > 0 && (h->loss == DIB_LOSS_EXTERNAL || h->loss == DIB_LOSS_INFONCE))
    return fail("dib_set_metrics: the external and InfoNCE losses take no compiled metrics");
  DibMetricTable t;
  const bool sparse = h->loss == DIB_LOSS_SPARSE_CE_LOGITS;
  for (int k = 0; k < count; ++k) {
    const dib_metric_spec& m = specs[k];
    const std::string at = "dib_set_metrics: metric " + std::to_string(k) + ": ";
    if (m.kind < DIB_METRIC_MSE || m.kind > DIB_METRIC_CONFUSION) return fail(at + "unknown kind");
    const bool label_kind = m.kind == DIB_METRIC_SPARSE_CATEGORICAL_ACCURACY || m.kind == DIB_METRIC_SPARSE_CATEGORICAL_CROSSENTROPY;
    if (label_kind != sparse)
      return fail(at + (sparse ? "the sparse categorical loss's targets are class labels: only the sparse kinds read them"
                               : "the sparse kinds need the sparse categorical loss's class-label targets"));
    t.kind[k] = m.kind; t.weighted[k] = m.weighted ? 1 : 0; t.from_logits[k] = m.from_logits ? 1 : 0;
    t.threshold[k] = m.threshold; t.off[k] = t.tail; t.boff[k] = 0; t.nthr[k] = 0;
    if (m.kind == DIB_METRIC_CONFUSION) {
      if (h->out != 1) return fail(at + "confusion metrics need output_dimensionality 1");
      if (m.num_thresholds < 1 || t.buckets + m.num_thresholds + 1 > DIB_MAX_METRIC_BUCKETS)
        return fail(at + "num_thresholds must be >= 1, with at most DIB_MAX_METRIC_BUCKETS buckets over all confusion metrics");
      t.nthr[k] = m.num_thresholds; t.boff[k] = t.buckets;
      t.buckets += m.num_thresholds + 1;
      t.tail += 2 * (m.num_thresholds + 1);
      if (m.from_logits) t.sigmoid = true;
    } else {
      t.tail += 2;
    }
  }
  t.count = count;
  DIB_CUDA_OK(dib_metrics_prepare(t));
  if (count > 0 && !h->d_metric_counter) {
    DIB_CUDA_OK(cudaMalloc(&h->d_metric_counter, sizeof(unsigned int)));
    DIB_CUDA_OK(cudaMemset(h->d_metric_counter, 0, sizeof(unsigned int)));
    DIB_CUDA_OK(cudaDeviceSynchronize());
  }
  h->metrics = t;
  plan_metrics(h);
  return 0;
}

int dib_metrics_update_tail(const float* tail, double* acc, int32_t count, void* stream) {
  if (count < 0 || (count > 0 && (!tail || !acc))) return fail("dib_metrics_update_tail: bad arguments");
  DIB_CUDA_OK(dib_launch_metrics_update_tail(tail, acc, count, static_cast<cudaStream_t>(stream)));
  return 0;
}

int dib_class_weight_rows(const float* y, int64_t n, int32_t y_cols, const float* class_table, int32_t classes,
                          const float* sample_weight_or_null, float* out, void* stream) {
  if (n < 0 || classes < 1 || y_cols < 0) return fail("dib_class_weight_rows: n >= 0, classes >= 1 and y_cols >= 0 are required");
  if (n > 0 && (!y || !class_table || !out)) return fail("dib_class_weight_rows: null y / class_table / out");
  DIB_CUDA_OK(dib_launch_class_weight_rows(y, n, y_cols, class_table, classes, sample_weight_or_null, out,
                                           static_cast<cudaStream_t>(stream)));
  return 0;
}

int dib_adam_step(float* params, const float* grads, float* m, float* v, int64_t count, const float* lr_dev,
                  int32_t* step_dev, float beta_1, float beta_2, float epsilon, void* stream) {
  if (!params || !grads || !m || !v || !lr_dev || !step_dev) return fail("dib_adam_step: null pointer");
  if (count < 0) return fail("dib_adam_step: negative count");
  DIB_CUDA_OK(dib_launch_adam(params, grads, m, v, count, lr_dev, step_dev, beta_1, beta_2, epsilon,
                              static_cast<cudaStream_t>(stream)));
  return 0;
}

int dib_optimizer_step(int32_t kind, float* params, const float* grads, float* slot1, float* slot2, int64_t count,
                       const float* lr_dev, int32_t* step_dev, float hyper0, float hyper1, float hyper2, void* stream) {
  if (kind < 0 || kind > 1 || !params || !grads || !lr_dev || !step_dev || count < 0 || (kind == 1 && (!slot1 || !slot2)) ||
      (kind == 0 && hyper0 != 0.f && !slot1))
    return fail("dib_optimizer_step: bad arguments");
  DIB_CUDA_OK(dib_launch_optimizer(kind, params, grads, slot1, slot2, count, lr_dev, step_dev, hyper0, hyper1, hyper2,
                                   static_cast<cudaStream_t>(stream)));
  return 0;
}

int dib_integration_forward(dib_model* h, const float* params, const float* emb, int64_t n, float* out_pred,
                            void* workspace, void* stream) {
  if (check_call(h, params, emb, n, workspace) || check_sets(h, n)) return 1;
  if (!out_pred) return fail("dib_integration_forward: null output");
  if (n == 0) return 0;
  Ctx c{h, params, static_cast<float*>(workspace), static_cast<cudaStream_t>(stream), (int)n};
  const int FE = h->F * h->E;
  if (tf32_shadow(c)) return 1;
  if (h->st) {                 // emb [n, Ls, E] (E is a multiple of 4: no padded columns) through the blocks and the mean
    const Ctx cr = particle_rows(c, NoiseKey{}).c;
    if (is_tc(h)) DIB_CUDA_OK(dib_launch_round_copy(emb, c.ws + h->emb.off, (int64_t)cr.n * FE, c.st));
    else DIB_CUDA_OK(dib_launch_copy2d(emb, FE, c.ws + h->emb.off, h->emb.ld, FE, cr.n, c.st));
    if (cr.sizes) DIB_CUDA_OK(dib_launch_zero_pad_rows(c.ws + h->emb.off, h->emb.ld, cr.n, h->Ls, cr.sizes, c.st));
    if (forward_set_blocks(cr)) return 1;
  } else {
    DIB_CUDA_OK(dib_launch_copy2d(emb, FE, c.ws + h->emb.off, h->emb.ld, FE, n, c.st));
    if (h->emb.ld > FE)          // zero the padded operand columns
      DIB_CUDA_OK(cudaMemset2DAsync(c.ws + h->emb.off + FE, sizeof(float) * h->emb.ld, 0, sizeof(float) * (h->emb.ld - FE), (size_t)n, c.st));
  }
  if (stack_forward(c, h->int_stack, 0, 1)) return 1;
  DIB_CUDA_OK(dib_launch_copy2d(c.ws + h->pred.off, h->pred.ld, out_pred, h->out, h->out, n, c.st));
  return 0;
}

int dib_output_encoder_forward(dib_model* h, const float* params, const float* y, int64_t n, float* out, void* workspace, void* stream) {
  if (check_call(h, params, y, n, workspace)) return 1;
  if (!infonce(h)) return fail("dib_output_encoder_forward: the model has no output encoder (loss is not DIB_LOSS_INFONCE)");
  if (!out) return fail("dib_output_encoder_forward: null output");
  if (n == 0) return 0;
  Ctx c{h, params, static_cast<float*>(workspace), static_cast<cudaStream_t>(stream), (int)n};
  if (tf32_shadow(c) || forward_output_encoder(c, y)) return 1;
  DIB_CUDA_OK(dib_launch_copy2d(c.ws + h->y_out.off, h->y_out.ld, out, h->out, h->out, n, c.st));
  return 0;
}

int dib_positional_encoding(const float* x, int64_t n, int32_t d, int32_t number_frequencies, float* out, void* stream) {
  if ((!x || !out) && n > 0) return fail("dib_positional_encoding: null pointer");
  if (n < 0 || d < 1 || number_frequencies < 1 || number_frequencies > 31) return fail("dib_positional_encoding: bad sizes");
  DIB_CUDA_OK(dib_launch_pe_plain(x, n, d, number_frequencies, out, static_cast<cudaStream_t>(stream)));
  return 0;
}

int dib_metrics_update_ex(const float* stats, const float* beta_dev, float* acc, int32_t number_features,
                          float kl_loss_exponent, float kl_loss_scale, void* stream) {
  if (!stats || !beta_dev || !acc || number_features < 1) return fail("dib_metrics_update: bad arguments");
  DIB_CUDA_OK(dib_launch_metrics_update(stats, beta_dev, acc, number_features, kl_loss_exponent == 0.f ? 1.f : kl_loss_exponent,
                                        kl_loss_scale == 0.f ? 1.f : kl_loss_scale, static_cast<cudaStream_t>(stream)));
  return 0;
}

int dib_metrics_update(const float* stats, const float* beta_dev, float* acc, int32_t number_features, void* stream) {
  return dib_metrics_update_ex(stats, beta_dev, acc, number_features, 1.f, 1.f, stream);
}

int dib_encoders_forward(dib_model* h, const float* params, const float* x, int64_t n, const float* eps, uint64_t seed,
                         uint32_t step, uint64_t sample_offset, float* out_emb, float* out_stats, void* workspace, void* stream) {
  if (check_call(h, params, x, n, workspace)) return 1;
  if (h->st) return fail("dib_encoders_forward: a set-transformer model trains its encoder through dib_train_step");
  if (!out_emb || !out_stats) return fail("dib_encoders_forward: out_emb and out_stats are required");
  Ctx c{h, params, static_cast<float*>(workspace), static_cast<cudaStream_t>(stream), (int)n};
  if (n == 0) { DIB_CUDA_OK(cudaMemsetAsync(out_stats, 0, sizeof(float) * (h->F + 3), c.st)); return 0; }
  return run_forward(c, x, nullptr, NoiseKey{eps, seed, step, sample_offset, false}, 0.f, nullptr, out_emb, out_stats, true);
}

int dib_encoders_backward(dib_model* h, const float* params, const float* x, const float* d_emb, int64_t n,
                          const float* beta_dev, float inv_global_batch, const float* eps, uint64_t seed, uint32_t step,
                          uint64_t sample_offset, float* grads_flat, float* out_stats, void* workspace, void* stream) {
  if (check_call(h, params, x, n, workspace)) return 1;
  if (h->st) return fail("dib_encoders_backward: a set-transformer model trains its encoder through dib_train_step");
  if ((!d_emb && n > 0) || !beta_dev || !grads_flat || !out_stats)
    return fail("dib_encoders_backward: d_emb, beta_dev, grads_flat and out_stats are required");
  Ctx c{h, params, static_cast<float*>(workspace), static_cast<cudaStream_t>(stream), (int)n};
  DIB_CUDA_OK(cudaMemsetAsync(grads_flat, 0, sizeof(float) * h->P, c.st));
  if (n == 0) { DIB_CUDA_OK(cudaMemsetAsync(out_stats, 0, sizeof(float) * (h->F + 3), c.st)); return 0; }
  // the forward is recomputed here (training mode keeps what the backward needs); user_emb is not needed again
  const NoiseKey nk{eps, seed, step, sample_offset, true};
  if (run_forward(c, x, nullptr, nk, inv_global_batch, nullptr, nullptr, out_stats, true)) return 1;
  const float* bw = beta_dev;
  if (ib_weight(c, beta_dev, out_stats, inv_global_batch, &bw)) return 1;
  int nrows = 0;
  if (backward_encoders(c, x, nk, d_emb, h->F * h->E, nullptr, bw, inv_global_batch, batch_split(n), &nrows)) return 1;
  DIB_CUDA_OK(dib_launch_reduce_partials(c.ws + h->part_off, h->Pp, nrows, h->intW[0], grads_flat, c.st));
  return 0;
}

int dib_mi_sandwich_bounds(const float* mu_logvar, int64_t n, int32_t embedding_dimension, const float* eps, uint64_t seed,
                           uint32_t step, float* row_scratch, float* out_lower_upper, void* stream) {
  if (!mu_logvar || !row_scratch || !out_lower_upper || n < 1 || n > 0x7fffffffll || embedding_dimension < 1)
    return fail("dib_mi_sandwich_bounds: bad arguments");
  DIB_CUDA_OK(dib_launch_mi_sandwich(mu_logvar, n, embedding_dimension, eps, seed, step, row_scratch, out_lower_upper,
                                     static_cast<cudaStream_t>(stream)));
  return 0;
}

int dib_mi_sandwich_bounds_batched(const float* mu_logvar, int32_t groups, int64_t n, int32_t embedding_dimension, const float* eps,
                                   uint64_t seed, int32_t batches_per_feature, double* row_scratch, double* out_lower_upper,
                                   void* stream) {
  if (!mu_logvar || !row_scratch || !out_lower_upper || groups < 1 || groups > 65535 || n < 1 || n > 0x7fffffffll ||
      embedding_dimension < 1 || embedding_dimension > 64 || batches_per_feature < 1)
    return fail("dib_mi_sandwich_bounds_batched: bad arguments (1 <= groups <= 65535, 1 <= E <= 64)");
  DIB_CUDA_OK(dib_launch_mi_sandwich_batched(mu_logvar, groups, n, embedding_dimension, eps, seed, batches_per_feature,
                                             row_scratch, out_lower_upper, static_cast<cudaStream_t>(stream)));
  return 0;
}

int dib_mi_bounds_at_probes(const float* probe_mu_logvar, int64_t m, const float* data_mu_logvar,
                            const int64_t* batch_offsets, int32_t batches, int32_t embedding_dimension, const float* eps,
                            uint64_t seed, void* scratch, double* out_lower_upper, void* stream) {
  if (!probe_mu_logvar || !data_mu_logvar || !batch_offsets || !scratch || !out_lower_upper)
    return fail("dib_mi_bounds_at_probes: null pointer");
  if (m < 1 || m > 0x7fffffffll || batches < 1 || batches > 65535 || embedding_dimension < 1 || embedding_dimension > 128)
    return fail("dib_mi_bounds_at_probes: bad arguments (1 <= m < 2^31, 1 <= batches <= 65535, 1 <= E <= 128)");
  if (reinterpret_cast<uintptr_t>(scratch) % 256 != 0) return fail("dib_mi_bounds_at_probes: scratch must be 256-byte aligned");
  DIB_CUDA_OK(dib_launch_mi_probes(probe_mu_logvar, m, data_mu_logvar, batch_offsets, batches, embedding_dimension, eps, seed,
                                   scratch, out_lower_upper, static_cast<cudaStream_t>(stream)));
  return 0;
}

size_t dib_mi_bounds_at_probes_scratch_bytes(int64_t m, int64_t data_rows, int32_t batches, int32_t embedding_dimension) {
  if (m < 0 || data_rows < 0 || batches < 0 || embedding_dimension < 1) return 0;
  return dib_mi_probes_scratch_bytes(m, data_rows, batches, embedding_dimension);
}

int dib_bhattacharyya(const float* mu_logvar, int64_t n, int32_t embedding_dimension, float* out_dist,
                      float* out_compression, void* stream) {
  if (!mu_logvar || n < 0 || embedding_dimension < 1) return fail("dib_bhattacharyya: bad arguments");
  const int64_t ld = 2 * (int64_t)embedding_dimension;
  DIB_CUDA_OK(dib_launch_pairwise_gauss(0, mu_logvar, ld, 0, n, mu_logvar, ld, 0, n, embedding_dimension, 1, out_dist,
                                        out_compression, static_cast<cudaStream_t>(stream)));
  return 0;
}

int dib_pairwise_gaussian(int32_t kind, const float* mu_logvar_1, int64_t n, const float* mu_logvar_2, int64_t m,
                          int32_t embedding_dimension, float* out, float* out_exp_neg, void* stream) {
  if ((kind != 0 && kind != 1) || n < 0 || m < 0 || embedding_dimension < 1 ||
      ((!mu_logvar_1 || !mu_logvar_2) && n > 0 && m > 0))
    return fail("dib_pairwise_gaussian: bad arguments");
  const int64_t ld = 2 * (int64_t)embedding_dimension;
  DIB_CUDA_OK(dib_launch_pairwise_gauss(kind, mu_logvar_1, ld, 0, n, mu_logvar_2, ld, 0, m, embedding_dimension, 1, out,
                                        out_exp_neg, static_cast<cudaStream_t>(stream)));
  return 0;
}

int dib_scaled_similarity(int32_t kind, const float* e1, int64_t n, const float* e2, int64_t m, int32_t d, float temperature,
                          float* out, void* stream) {
  if (kind < 0 || kind > 4 || n < 0 || m < 0 || d < 1 || !(temperature > 0.f) || ((!e1 || !e2 || !out) && n > 0 && m > 0))
    return fail("dib_scaled_similarity: bad arguments");
  DIB_CUDA_OK(dib_launch_similarity(kind, e1, n, e2, m, d, temperature, out, static_cast<cudaStream_t>(stream)));
  return 0;
}

int dib_infonce_head(int32_t kind, const float* e1, const float* e2, int64_t n, int32_t d, float temperature, float* scratch,
                     float* out_loss, float* d_e1, float* d_e2, void* stream) {
  if (kind < 0 || kind > 4 || n < 1 || n > 32768 || d < 1 || d > 512 || !(temperature > 0.f) || !e1 || !e2 || !scratch ||
      !out_loss)
    return fail("dib_infonce_head: bad arguments (1 <= n <= 32768, 1 <= d <= 512, temperature > 0)");
  DIB_CUDA_OK(dib_launch_infonce_head(kind, e1, e2, n, d, temperature, scratch, out_loss, d_e1, d_e2,
                                      static_cast<cudaStream_t>(stream)));
  return 0;
}

int dib_compression_matrices(dib_model* h, const float* params, const float* x, int64_t n_total, const int32_t* row_index,
                             int64_t n, float* out_mu_logvar, float* out_dist, float* out_compression, void* workspace,
                             void* stream) {
  if (check_call(h, params, x, n, workspace)) return 1;
  if (n_total < 0 || (!row_index && n > n_total) || (row_index && n > 0 && n_total < 1))
    return fail("dib_compression_matrices: rows out of range");
  if (n == 0) return 0;
  Ctx c{h, params, static_cast<float*>(workspace), static_cast<cudaStream_t>(stream), (int)n};
  if (tf32_shadow(c)) return 1;
  // all F encoders as ONE grouped problem per layer (the reference loops over features in Python, visualization.py:14-35)
  if (encode_all(c, x, h->D, -1, row_index, n_total)) return 1;
  const float* eo = c.ws + h->enc_out.off;
  if (out_mu_logvar)
    for (int f = 0; f < h->F; ++f)
      DIB_CUDA_OK(dib_launch_copy2d(eo + f * h->enc_out.feat_stride, h->enc_out.ld, out_mu_logvar + (int64_t)f * n * 2 * h->E,
                                    2 * h->E, 2 * h->E, n, c.st));
  if (out_dist || out_compression)
    DIB_CUDA_OK(dib_launch_pairwise_gauss(0, eo, h->enc_out.ld, h->enc_out.feat_stride, n, eo, h->enc_out.ld,
                                          h->enc_out.feat_stride, n, h->E, h->F, out_dist, out_compression, c.st));
  return 0;
}

}  // extern "C"
