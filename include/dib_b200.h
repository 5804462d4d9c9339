/* dib_b200.h -- C ABI of the H100-native Distributed-IB training engine.
 *
 * The reference (distributed-information-bottleneck.github.io) has no FFI/plugin interface: its
 * hot path is a tf.keras Model whose arithmetic executes inside TensorFlow.  Each entry point
 * below therefore names the reference *Python* interface it replaces (paths relative to the
 * reference root).  The PyTorch host shim (package dib_b200) binds these with ctypes and
 * reproduces the DistributedIBNet / compile / fit / callback surface on top of them;
 * INTEGRATION.md shows the stub a maintainer of the reference would add.
 *
 * Conventions
 *   - every pointer named *_dev / params / grads / x / y / eps / workspace is DEVICE memory owned by
 *     the caller (PyTorch tensors in the shim); the library never allocates user-visible memory.
 *     The only allocation it makes is a few KB of layer-descriptor tables inside dib_create.
 *   - every compute call is asynchronous on the caller's cudaStream_t (passed as void*), performs no
 *     host synchronisation and no allocation, and is CUDA-Graph capturable: beta, learning rate and
 *     the Adam step counter are read from device scalars.
 *   - return value: 0 = ok, non-zero = error (see dib_last_error()); no C++ exception crosses.
 *   - a handle is not thread-safe; use one host thread per handle (the reference is single-threaded).
 *   - all tensors are fp32, row-major.  Parameters live in ONE flat fp32 buffer; per feature
 *     (W1,b1,W2,b2,...,W_out,b_out) then the integration layers, kernels in Keras [in,out]
 *     orientation (tf.keras.layers.Dense, models.py:76-77,82-83).
 *   - sums, not means: statistics are returned as SUMS over the local samples so that data-parallel
 *     ranks combine them (and the gradients) with one all-reduce(sum); gradients are already scaled
 *     by inv_global_batch.
 */
#ifndef DIB_B200_H_
#define DIB_B200_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

/* 3 appended the InfoNCE fields to dib_config, 4 the integration-network fields, 5 variable_set_sizes; dib_create still accepts
 * abi_version 2, 3 and 4 structs and reads only their prefix. */
#define DIB_ABI_VERSION 5

/* largest set_size of a set transformer with variable_set_sizes (fixed-size sets: 64) */
#define DIB_MAX_VARIABLE_SET_SIZE 256

/* activation_fn strings accepted by tf.keras.layers.Dense in the reference's call sites
 * (train.py:37 'relu', nb-radial 'tanh', nb-bool LeakyReLU, None). */
enum dib_activation {
  DIB_ACT_LINEAR = 0, DIB_ACT_RELU = 1, DIB_ACT_TANH = 2, DIB_ACT_LEAKY_RELU = 3,
  DIB_ACT_SIGMOID = 4, DIB_ACT_ELU = 5
};

/* compiled losses used by the reference's datasets (data.py:65, data.py:343, data.py:129). */
enum dib_loss {
  DIB_LOSS_BCE_LOGITS = 0,       /* tf.keras.losses.BinaryCrossentropy(from_logits=True)            */
  /* tf.keras.losses.SparseCategoricalCrossentropy(from_logits=True).  As TensorFlow on a GPU: a label t names class (int)t
   * (truncation) when -1 < t < output_dimensionality; any other label (NaN included) gives a NaN loss and a NaN d loss / d z
   * for its row, and no accuracy hit.  An accuracy hit is float(argmax z) == t. */
  DIB_LOSS_SPARSE_CE_LOGITS = 1,
  DIB_LOSS_MSE = 2,
  /* NEXT ROW f3 -- custom training steps (GradientTape loops: train.py:201-220 InfoNCE, nb-bool cell 6, nb-particle
   * cell 7): the CALLER owns the task loss.  dib_forward returns the predictions; in dib_train_step the `y` argument
   * is reinterpreted as d(task loss)/d(predictions) [n, out], already carrying the caller's batch-mean scaling (it is
   * NOT multiplied by inv_global_batch; the beta*KL term still is).  Task-loss and accuracy statistics are 0. */
  DIB_LOSS_EXTERNAL = 3,
  /* tf.keras.losses.BinaryCrossentropy() on PROBABILITIES (from_logits=False, the Keras default; use with
   * output_activation_fn = sigmoid): -[y log(p~ + eps) + (1-y) log(1 - p~ + eps)], p~ = clip(p, eps, 1-eps), eps = 1e-7
   * (keras.backend.binary_crossentropy); the gradient is zero where p is clipped. */
  DIB_LOSS_BCE_PROBS = 4,
  /* the InfoNCE path of train.py:180-289 (--infonce_loss; data.py:131's double pendulum): the model is trained together
   * with an OUTPUT ENCODER for y (train.py:186-193: positional encoding as the model's, Dense(h, activation_fn) for every
   * width of y_encoder_architecture, then a linear Dense(output_dimensionality)), whose variables follow the model's in the
   * flat buffer (train.py:198).  y is the raw [n, y_dimensionality] target.  Task loss = the symmetric InfoNCE of
   * train.py:203-213 over the [n, n] similarity matrix of (pred, output_encoder(y)), computed by streaming kernels whose
   * memory is linear in n (the matrix is never stored).  It couples every row of the batch, so n is the whole batch:
   * inv_global_batch scales only the beta*KL term.  Stats: task-loss slot = n * loss, accuracy slot 0.
   * Needs abi_version >= 3, output_activation_fn = DIB_ACT_LINEAR and output_dimensionality <= 512. */
  DIB_LOSS_INFONCE = 5
};

/* Per-sample weights of the compiled loss (Keras fit / evaluate / train_on_batch sample_weight=, class_weight=), reduction
 * SUM_OVER_BATCH_SIZE: task loss = sum_i w_i l_i / n with n the (global) batch size, not sum w; d loss / d z_i is w_i times
 * the unweighted value; the beta*KL term and the accuracy statistic are not weighted.  The task-loss slot of the stats holds
 * sum_i w_i l_i.  Declared after dib_model below:
 *
 *   int dib_set_sample_weights_device(dib_model* h, const float* w_dev);
 *     binds w_dev (DEVICE memory, 4-byte aligned): the fp32 weights of the n rows (sets, for a set transformer) of the following
 *     dib_forward and dib_train_step calls of this handle (data parallel: this rank's shard).  The loss kernels read it on the
 *     stream, so one captured graph serves every weight vector written into the buffer.  NULL (the default) = unweighted.  The
 *     caller checks that the weights are finite and >= 0.  Fails on DIB_LOSS_EXTERNAL and DIB_LOSS_INFONCE handles.
 *
 *   int dib_class_weight_rows(const float* y, int64_t n, int32_t y_cols, const float* class_table, int32_t classes,
 *                             const float* sample_weight_or_null, float* out, void* stream);
 *     Keras' class_weight map (_make_class_weight_map_fn) on the device: the class of row i is argmax_j y[i, j] when
 *     y_cols > 1, else y[i] cast to an integer (truncating); out[i] = class_table[class] * sample_weight[i] (the product only
 *     when sample_weight_or_null is given).  A class outside [0, classes) gives NaN, which the caller must not bind.  y, the
 *     table, the sample weights and out are DEVICE memory; y_cols = 0 or 1 reads y as [n]. */

/* Compiled Keras metrics beyond metrics=['accuracy'] (Keras 2 semantics; see dib_set_metrics below).  Each metric adds sums
 * to a METRIC TAIL behind the F + 3 statistics, so dib_stats_count = F + 3 + M; every entry is a sum over rows, so the
 * all-reduce of [grads || stats] that data parallelism already does also sums the tail.  m_i is the row's value averaged over
 * the outputs, w_i its sample weight (1 unless the metric is weighted and weights are bound):
 *   mean metrics, 2 floats: [ sum_i w_i m_i | sum_i w_i ]   (epoch value = sum w m / sum w)
 *     DIB_METRIC_MSE (z - y)^2;  DIB_METRIC_MAE |z - y|;  DIB_METRIC_BINARY_ACCURACY [(z > threshold) == y];
 *     DIB_METRIC_SPARSE_CATEGORICAL_ACCURACY [argmax z == y];  DIB_METRIC_BINARY_CROSSENTROPY (from_logits: the logistic
 *     loss of z; else keras.backend.binary_crossentropy: p clipped to [1e-7, 1 - 1e-7], -(y log(p + 1e-7) + (1-y) log(1 - p
 *     + 1e-7)));  DIB_METRIC_SPARSE_CATEGORICAL_CROSSENTROPY (from_logits: logsumexp z - z_y; else -log(p~_y / sum_j p~_j),
 *     p~ = p clipped to [1e-7, 1 - 1e-7]).  The two sparse kinds need y [n] class labels, the others y [n, out].
 *   DIB_METRIC_CONFUSION (out = 1), 2 (T + 1) floats: [ neg[0..T] | pos[0..T] ], the summed w of the rows with y == 0 (neg)
 *     and y != 0 (pos) whose p (sigmoid(z) with from_logits, else z) exceeds exactly b of the T float32 thresholds
 *     (p > t strictly).  T >= 2: Keras' AUC table {-1e-7, 1/(T-1), ..., (T-2)/(T-1), 1 + 1e-7}; T == 1: {threshold}
 *     (Precision / Recall).  TP(t_j) = sum_{b > j} pos[b], FP(t_j) = sum_{b > j} neg[b], FN and TN the rest. */
enum dib_metric_kind {
  DIB_METRIC_MSE = 0,
  DIB_METRIC_MAE = 1,
  DIB_METRIC_BINARY_ACCURACY = 2,
  DIB_METRIC_SPARSE_CATEGORICAL_ACCURACY = 3,
  DIB_METRIC_BINARY_CROSSENTROPY = 4,
  DIB_METRIC_SPARSE_CATEGORICAL_CROSSENTROPY = 5,
  DIB_METRIC_CONFUSION = 6
};
#define DIB_MAX_METRICS 16
#define DIB_MAX_METRIC_BUCKETS 2048      /* sum over the confusion metrics of (num_thresholds + 1) */

typedef struct dib_metric_spec {
  int32_t kind;             /* dib_metric_kind */
  int32_t weighted;         /* 1: w_i = the bound sample weight (dib_set_sample_weights_device), 0: w_i = 1 */
  int32_t from_logits;      /* crossentropy and confusion metrics: z is a logit */
  int32_t num_thresholds;   /* DIB_METRIC_CONFUSION: T (1 .. DIB_MAX_METRIC_BUCKETS - 1); otherwise 0 */
  float threshold;          /* DIB_METRIC_BINARY_ACCURACY, and DIB_METRIC_CONFUSION with T == 1 */
} dib_metric_spec;

/* arithmetic of the dense contractions; everything else (PE, exp, KL, loss, Adam, reductions) is fp32 in every mode
 * and all tensor-core modes accumulate in fp32 (wgmma register accumulators).
 *   FP32: CUDA-core FMA -- the exact parity path (the reference's tf.keras fp32 graph on a CPU).
 *   TF32: tf32 wgmma on fp32 storage (10-bit mantissa, 8-bit exponent operands, rounded not truncated):
 *         what stock TensorFlow does to an fp32 model on a tensor-core GPU.  Unfused grouped GEMMs.
 *   FP16: f16 wgmma on fp16 operands (10-bit mantissa like TF32 but a 5-bit exponent: |value| <= 65504,
 *         saturating conversions, gradients carried under a power-of-two loss scale) -- the fused per-feature encoder
 *         kernels and the 16-bit integration path; shapes outside their envelope run on the TF32 kernels.
 *   BF16: the same fused kernels on bf16 operands (7-bit mantissa, fp32's exponent range).
 * dib_model_info() reports which kernel family a handle actually selected. */
enum dib_precision { DIB_PREC_FP32 = 0, DIB_PREC_TF32 = 1, DIB_PREC_BF16 = 2, DIB_PREC_FP16 = 3 };

/* feature encoders: the per-feature MLP of models.py:72-78, or nb-bool cell 4's SimpleEncoder -- two trainable (1,1)
 * constants per feature, output concat([x * mu_scaling, ones_like(x) * logvar]) (needs d_i == E, no positional encoding;
 * flat parameter order per feature: mu_scaling, logvar; feature_encoder_architecture is ignored). */
enum dib_encoder_kind { DIB_ENCODER_MLP = 0, DIB_ENCODER_SIMPLE = 1 };

/* integration networks: the Dense stack of models.py:81-84, or the per-particle set transformer of nb-particle cell 8.
 * DIB_INTEGRATION_SET_TRANSFORMER: number_features == 1 and x is [n, set_size, d] -- n counts SETS of set_size particles,
 * y is [n, out], max_batch counts sets (the workspace holds max_batch * set_size particle rows).  The one feature encoder runs
 * with shared weights on every particle; its embeddings [n, L, E] pass number_attention_blocks blocks of
 *   H = LayerNorm(x + MultiHeadAttention(number_heads, key_dim)(x, x, x)),  x' = LayerNorm(H + FF(H))
 * (Keras 2 MultiHeadAttention without dropout or mask; FF = Dense(ff_architecture[j], ff_activation_fn) for every j, the
 * last width equal to E; LayerNorm with layer_norm_epsilon, biased variance), then the mean over the particles feeds the Dense
 * head integration_network_architecture (activation_fn) -> output_dimensionality (output_activation_fn).
 * Flat parameter order: the encoder, then per block q kernel [E, h*dk], q bias [h*dk], k, k bias, v, v bias, output kernel
 * [h*dk, E], output bias [E], LN1 gamma, LN1 beta, the FF kernels and biases, LN2 gamma, LN2 beta; then the head.
 * Statistics: the KL slot sums over sets, particles and dims; inv_global_batch is 1 / (global number of sets); the noise of
 * particle p of set s is keyed by the global particle row (sample_offset + s) * set_size + p.
 * Needs set_size in [1, 64], key_dim in [1, 128], number_heads * key_dim and E multiples of 4, E <= 128, max_batch <= 65535,
 * no dropout, and a loss other than DIB_LOSS_SPARSE_CE_LOGITS / DIB_LOSS_INFONCE.  The attention core and the LayerNorms are
 * fp32 CUDA-core kernels in every precision; FP16 / BF16 run every dense layer on the TF32 kernels.
 * Variable set sizes (abi_version >= 5, variable_set_sizes = 1; nb-particle's ragged neighbourhoods): set_size is the largest
 * set Lmax, in [1, DIB_MAX_VARIABLE_SET_SIZE].  x stays [n, Lmax, d], each set padded to Lmax rows, and set s has l_s real
 * particles, 1 <= l_s <= Lmax, given by dib_set_set_sizes_device.  Per set, loss, KL, prediction and gradients are those of the
 * fixed-size model with set_size = l_s on the real particles: keys p >= l_s are masked out of every softmax (Keras 2
 * MultiHeadAttention with attention_mask), the mean runs over the l_s real rows, and the KL slot sums over real particles only.
 * Padding rows are zeroed before the encoder and get u = 0 and zero gradients: their content, NaN included, changes nothing.
 * Noise stays keyed by the padded row (sample_offset + s) * set_size + p.  The attention runs on key-tiled kernels whose
 * shared memory does not depend on Lmax and whose work follows sum_s l_s^2; the dense layers still run on all n * Lmax rows.
 * The workspace stays linear in max_batch * set_size. */
enum dib_integration_kind { DIB_INTEGRATION_MLP = 0, DIB_INTEGRATION_SET_TRANSFORMER = 1 };

/* Mirrors the constructor of models.DistributedIBNet (models.py:56-66). */
typedef struct dib_config {
  int32_t abi_version;               /* DIB_ABI_VERSION */
  int32_t number_features;           /* len(feature_dimensionalities)            models.py:69 */
  const int32_t* feature_dimensionalities;     /* [number_features]             models.py:68 */
  int32_t number_encoder_layers;     /* len(feature_encoder_architecture) */
  const int32_t* feature_encoder_architecture; /* hidden widths                  models.py:76 */
  int32_t number_integration_layers; /* len(integration_network_architecture) */
  const int32_t* integration_network_architecture; /*                            models.py:82 */
  int32_t output_dimensionality;     /*                                          models.py:83 */
  int32_t use_positional_encoding;   /*                                          models.py:74 */
  int32_t number_positional_encoding_frequencies; /* n -> frequencies 2^1..2^(n-1), models.py:70 */
  int32_t activation_fn;             /* enum dib_activation */
  float   leaky_relu_alpha;          /* slope for DIB_ACT_LEAKY_RELU */
  int32_t feature_embedding_dimension; /* E                                      models.py:64 */
  int32_t output_activation_fn;      /* enum dib_activation                      models.py:83 */
  int32_t loss;                      /* enum dib_loss (model.compile(loss=...), train.py:138-142) */
  int32_t precision;                 /* enum dib_precision */
  int64_t max_batch;                 /* largest n any call will pass (sizes the workspace) */
  /* ---- custom-step variants of the same front end (NEXT ROW f3); zero-initialised fields give models.py ---- */
  float   logvar_offset;             /* constant added to every encoder's log-variance before sampling / KL / any output
                                        (nb-particle cell 8: embs_logvars + logvar_initialization, -3 there) */
  float   kl_loss_exponent;          /* nonlinear IB (nb-chaos cell 10): loss_IB = beta * kl_loss_scale * (sum_i KL_i)^exponent; */
  float   kl_loss_scale;             /*   0 or 1 / 0 or 1 = the linear beta * sum_i KL_i of models.py:118 */
  int32_t encoder_kind;              /* enum dib_encoder_kind */
  float   dropout_rate;              /* nb-radial cell 5: tf.keras.layers.Dropout(rate) after every hidden Dense of the feature
                                        encoders, active in dib_train_step only (Keras training=True); masks from the Philox
                                        stream (oracle/philox.py :: dropout_keep).  Encoders then run on the unfused kernels. */
  /* ---- abi_version >= 3: the output encoder and loss of DIB_LOSS_INFONCE (ignored for every other loss) ---- */
  int32_t y_dimensionality;          /* width of y                                  train.py:186 */
  int32_t number_y_encoder_layers;   /* len(y_encoder_architecture) */
  const int32_t* y_encoder_architecture; /* hidden widths (--infonce_y_encoder_architecture)  train.py:189-190 */
  int32_t infonce_similarity;        /* 0 'l2sq' | 1 'l2' | 2 'l1' | 3 'linf' | 4 'cosine' (dib_scaled_similarity kinds) */
  float   infonce_temperature;       /* > 0                                          train.py:204 */
  /* ---- abi_version >= 4: the integration network (zero-initialised fields give models.py's Dense stack) ---- */
  int32_t integration_kind;          /* enum dib_integration_kind */
  int32_t set_size;                  /* L, particles per set (nb-particle clips every set to 50) */
  int32_t number_attention_blocks;   /* 6 in nb-particle cell 8 */
  int32_t number_heads;              /* 12 */
  int32_t key_dim;                   /* 128 */
  int32_t number_ff_layers;          /* len(ff_architecture) */
  const int32_t* ff_architecture;    /* [128, E] */
  int32_t ff_activation_fn;          /* enum dib_activation; relu on every FF layer in the notebook */
  float   layer_norm_epsilon;        /* 0 -> 1e-3 (the Keras default) */
  /* ---- abi_version >= 5 ---- */
  int32_t variable_set_sizes;        /* set transformer: 1 = sets of l_s <= set_size particles (dib_set_set_sizes_device) */
} dib_config;

typedef struct dib_model dib_model;

/* models.DistributedIBNet.__init__ (models.py:56-86).  Uses the current CUDA device. */
int dib_create(const dib_config* cfg, dib_model** out);
void dib_destroy(dib_model* h);

/* number of trainable parameters == sum over model.trainable_variables (train.py:198); with DIB_LOSS_INFONCE also the
 * output encoder's (all_trainable_variables = model vars + output_encoder vars, train.py:198). */
int64_t dib_param_count(const dib_model* h);

/* For every variable v (in flat order) its offset and shape: offsets[v], rows[v] (fan-in, or 0 for a
 * bias), cols[v].  Pass NULLs to query the number of variables (return value, negative on error). */
int dib_param_layout(const dib_model* h, int64_t* offsets, int32_t* rows, int32_t* cols, int32_t capacity);

/* bytes of scratch the caller must provide to forward / train_step / encode calls (linear in max_batch, DIB_LOSS_INFONCE
 * included).  The workspace pointer must be 256-byte
 * aligned and `params` 16-byte aligned (checked; cudaMalloc / torch allocations are). */
size_t dib_workspace_bytes(const dib_model* h);

/* number of floats in the statistics vector: [ sum_b KL_i (F) | sum_b task loss | sum_b accuracy | n ], followed by the
 * metric tail (M floats) when dib_set_metrics configured one: F + 3 + M, else F + 3 */
int32_t dib_stats_count(const dib_model* h);

/* DistributedIBNet.call (models.py:96-123) + compiled loss/metrics, no gradient: the validation pass of
 * Model.fit (train.py:157-166; noise is sampled in validation too, train.py:264-265).
 *   x [n, sum d_i]; y [n, out] (class index as float for sparse CE; DIB_LOSS_INFONCE: [n, y_dimensionality]) or NULL; eps [n, F, E] or NULL ->
 *   Philox4x32-10 keyed (seed, step, feature, sample_offset + row, dim), see oracle/philox.py;
 *   out_pred [n, out] or NULL; out_emb [n, F*E] or NULL; out_stats [dib_stats_count] (zeroed by the call). */
int dib_forward(dib_model* h, const float* params, const float* x, const float* y, int64_t n,
                const float* beta_dev, const float* eps, uint64_t seed, uint32_t step, uint64_t sample_offset,
                float* out_pred, float* out_emb, float* out_stats, void* workspace, void* stream);

/* model.feature_encoders[i](x_i) (models.py:79; consumers visualization.py:31, utils.py:38, nb-radial
 * StashEmbeddingsCallback): deterministic [n, d_i] -> [n, 2E] = (mu || logvar). */
int dib_encode_feature(dib_model* h, const float* params, int32_t feature, const float* x_i, int64_t n,
                       float* out_mu_logvar, void* workspace, void* stream);

/* One Keras train_step minus the optimizer: forward, loss = task + beta*sum_i KL_i (models.py:118),
 * reverse mode (GradientTape in Model.fit / nb-bool cell 6).  grads_flat [P] receives
 * d(loss)/d(params) * (n_local-sum scaled by inv_global_batch); out_stats as in dib_forward.
 * grads_flat and out_stats may be adjacent in one buffer so that one all-reduce covers both.
 * DIB_LOSS_INFONCE: forward, output-encoder forward, streaming InfoNCE (d pred, d output-encoder output), the model's backward
 * from d pred, the output encoder's backward into its slice of grads_flat -- one stream-ordered sequence, no host sync. */
int dib_train_step(dib_model* h, const float* params, const float* x, const float* y, int64_t n,
                   const float* beta_dev, float inv_global_batch,
                   const float* eps, uint64_t seed, uint32_t step, uint64_t sample_offset,
                   float* grads_flat, float* out_stats, void* workspace, void* stream);

/* dib_train_step of a DIB_LOSS_INFONCE model on one rank of a data-parallel group whose negatives are all rows of the GLOBAL
 * batch (train.py:203-219 on that batch: every rank computes the one-GPU loss and gradient).  The rank owns the n global rows
 * [row_offset, row_offset + n) of an n_global-row batch; the step runs as three phases with two exchanges between them that
 * the caller does (DESIGN.md section 7):
 *   1. dib_infonce_shard_forward (train.py:201-202, 209-210: model(x), output_encoder(y)): writes
 *      e_all[row_offset + i] = (e1_i || e2_i), e_all [n_global, 2 * output_dimensionality] row-major.
 *      -> the caller all-gathers e_all.
 *   2. dib_infonce_shard_lse (train.py:203-213): from all rows of e_all, the row log-sum-exps r_i of the own e1 rows and the
 *      column log-sum-exps c_j of the own e2 rows into lse_all[row_offset + i] = (r_i, c_i), lse_all [n_global, 2];
 *      out_stats [dib_stats_count] = KL sums of the own rows | sum_own (r_i + c_i - 2 s_ii) | 0 | n.
 *      -> the caller all-gathers lse_all.
 *   3. dib_infonce_shard_backward (train.py:216-220): d e1 of the own rows against all columns and d e2 of the own rows against
 *      all rows (weights (...) / n_global), the model's and the output encoder's backward, KL means over n_global:
 *      grads_flat [P] = this rank's share; the sum over ranks is the one-GPU gradient of the global batch.
 *      -> the caller all-reduces [grads || stats], then runs the optimizer.
 * Noise is keyed by sample_offset as in dib_train_step; dib_set_noise_step_device applies to phase 1 with training != 0 and to
 * phase 3 (phase 1 with training == 0 is the validation forward of dib_forward).  Phases 2 and 3 read what the phases before
 * them left in the workspace: run them in order on the same handle, workspace and inputs, with no other call on the handle in
 * between.  With row_offset = 0 and n = n_global the three phases are dib_train_step bit for bit.  Caller-owned buffers, the
 * caller's stream, no host sync.  Needs 1 <= n <= max_batch, row_offset + n <= n_global < 2^31, e_all and lse_all 16-byte
 * aligned. */
int dib_infonce_shard_forward(dib_model* h, const float* params, const float* x, const float* y, int64_t n, int32_t training,
                              const float* eps, uint64_t seed, uint32_t step, uint64_t sample_offset, float* e_all,
                              int64_t n_global, int64_t row_offset, void* workspace, void* stream);
int dib_infonce_shard_lse(dib_model* h, const float* e_all, int64_t n_global, int64_t row_offset, int64_t n, float* lse_all,
                          float* out_stats, void* workspace, void* stream);
int dib_infonce_shard_backward(dib_model* h, const float* params, const float* x, int64_t n, const float* beta_dev, const float* eps,
                               uint64_t seed, uint32_t step, uint64_t sample_offset, const float* e_all, const float* lse_all,
                               int64_t n_global, int64_t row_offset, float* grads_flat, void* workspace, void* stream);

/* NEXT ROW f3 -- encoder-only custom steps (nb-particle cell 8: a shared particle encoder feeding the caller's own
 * network, e.g. a set transformer; nb-chaos cell 10): the model's integration network is not used.
 *   dib_encoders_forward : x [n, sum d_i] -> out_emb [n, F*E] (u = mu + exp(logvar/2) eps) and out_stats (KL sums; loss = acc = 0).
 *   dib_encoders_backward: recomputes that forward, then reverse mode from d_emb [n, F*E] = d(caller's loss)/d(emb)
 *     (already carrying the caller's batch scaling) plus the IB term d(beta * scale * (sum KL)^p)/d(params) with KL means
 *     over inv_global_batch; grads_flat [P]: encoder entries written, integration-network entries zeroed.
 * A shared-weight encoder over a particle axis is F = 1 on n = B * particles rows with inv_global_batch = 1/B (KL summed
 * over particles, averaged over the batch). */
int dib_encoders_forward(dib_model* h, const float* params, const float* x, int64_t n, const float* eps, uint64_t seed,
                         uint32_t step, uint64_t sample_offset, float* out_emb, float* out_stats, void* workspace, void* stream);
int dib_encoders_backward(dib_model* h, const float* params, const float* x, const float* d_emb, int64_t n,
                          const float* beta_dev, float inv_global_batch, const float* eps, uint64_t seed, uint32_t step,
                          uint64_t sample_offset, float* grads_flat, float* out_stats, void* workspace, void* stream);

/* CUDA-Graph replay: a captured launch cannot carry a fresh by-value `step`, so the Philox step word may come from device
 * memory: when step_dev != NULL every later dib_train_step call of this handle uses step + *step_dev (dib_forward
 * and the encoder-only entry points keep the by-value step).  The caller owns the counter and advances it (on the stream)
 * between steps.  NULL restores the by-value behaviour. */
int dib_set_noise_step_device(dib_model* h, const uint32_t* step_dev);

/* Variable set sizes: set_sizes_dev is DEVICE memory holding the int32 sizes of the n local sets of the following dib_forward,
 * dib_train_step and dib_integration_forward calls of this handle (data parallel: the sizes of this rank's shard).  The kernels
 * read it on the stream, so one captured graph serves every size vector written into the buffer.  The caller checks
 * 1 <= size <= set_size (the library cannot without a sync): every kernel treats a size outside [1, set_size] as the nearest
 * bound, so such a set is computed, forward and backward alike, as a set of 1 or of set_size particles.  A variable-size handle
 * without bound sizes fails those calls; NULL unbinds.  Fails on a fixed-size handle. */
int dib_set_set_sizes_device(dib_model* h, const int32_t* set_sizes_dev);

/* per-sample weights of the compiled loss and Keras' class_weight map: see the comment after enum dib_loss */
int dib_set_sample_weights_device(dib_model* h, const float* w_dev);
int dib_class_weight_rows(const float* y, int64_t n, int32_t y_cols, const float* class_table, int32_t classes,
                          const float* sample_weight_or_null, float* out, void* stream);

/* Compiled metrics (see dib_metric_spec after enum dib_loss): specs[0 .. count) in order define the metric tail, which
 * dib_forward (with y) and dib_train_step write behind the F + 3 statistics.  The prediction is written to the workspace
 * (or to out_pred when given) and one launch after the loss reduces it with y and the weights into the tail, in a fixed
 * order (no float atomics: repeated calls and graph replays are bit-identical).  count = 0 removes the tail, and the calls
 * run exactly the launches they ran before.  Changes dib_stats_count and dib_workspace_bytes: query both after this call.
 * Fails (and changes nothing) on DIB_LOSS_EXTERNAL / DIB_LOSS_INFONCE handles, on a confusion metric with
 * output_dimensionality != 1, on the sparse kinds without DIB_LOSS_SPARSE_CE_LOGITS, on the other kinds with it, and
 * beyond DIB_MAX_METRICS / DIB_MAX_METRIC_BUCKETS.  The encoder-only entry points write the F + 3 statistics only. */
int dib_set_metrics(dib_model* h, const dib_metric_spec* specs, int32_t count);

/* epoch accumulation of a metric tail: acc[i] += (double)tail[i] for i < count (tail: the all-reduced floats behind the
 * F + 3 statistics; acc: float64 DEVICE memory the caller zeroes at the start of an epoch). */
int dib_metrics_update_tail(const float* tail, double* acc, int32_t count, void* stream);

/* tf.keras.optimizers.Adam dense update over the flat buffer (train.py:128-129, nb-radial Adam(lr)):
 *   t = *step_dev + 1 (the kernel increments *step_dev);  lr_t = lr*sqrt(1-b2^t)/(1-b1^t);
 *   m += (1-b1)(g-m); v += (1-b2)(g^2-v); w -= lr_t*m/(sqrt(v)+eps)   (eps outside the bias correction). */
int dib_adam_step(float* params, const float* grads, float* m, float* v, int64_t count,
                  const float* lr_dev, int32_t* step_dev, float beta_1, float beta_2, float epsilon,
                  void* stream);

/* the other optimizers tf.keras.optimizers.get(name) hands out (train.py:41,128); same device scalars as dib_adam_step.
 *   kind 0 SGD     : v = momentum * v - lr * g;  w += nesterov ? momentum * v - lr * g : v        (slot1 = v; slot2 unused)
 *   kind 1 RMSprop : ms = rho * ms + (1-rho) g^2;  mom = momentum * mom + lr * g / sqrt(ms + eps);  w -= mom   (TF ApplyRMSProp;
 *                    slot1 = ms, slot2 = mom)
 * hyper = {momentum, nesterov(0/1), 0} for SGD, {rho, momentum, epsilon} for RMSprop.  *step_dev is incremented. */
int dib_optimizer_step(int32_t kind, float* params, const float* grads, float* slot1, float* slot2, int64_t count,
                       const float* lr_dev, int32_t* step_dev, float hyper0, float hyper1, float hyper2, void* stream);

/* model.integration_network(emb) (models.py:84,122) as a stand-alone call: emb [n, F*E] -> out_pred [n, out] through the
 * Dense stack with the output activation, on the model's precision path (fp32 FMA / tf32 wgmma). */
int dib_integration_forward(dib_model* h, const float* params, const float* emb, int64_t n, float* out_pred,
                            void* workspace, void* stream);

/* output_encoder(y) of a DIB_LOSS_INFONCE model (train.py:186-193, deterministic): y [n, y_dimensionality] -> out [n, output_dimensionality]
 * on the model's precision path (fp32 FMA / tf32 wgmma). */
int dib_output_encoder_forward(dib_model* h, const float* params, const float* y, int64_t n, float* out, void* workspace, void* stream);

/* models.PositionalEncoding.call (models.py:12-23) as a stand-alone call: x [n, d] ->
 * out [n, d * number_frequencies] = concat([x] + [sin(2^k x) for k = 1 .. number_frequencies-1], -1), block-major. */
int dib_positional_encoding(const float* x, int64_t n, int32_t d, int32_t number_frequencies, float* out, void* stream);

/* Keras metric aggregation of one batch (Model.fit's Mean metrics; add_metric at models.py:115,121):
 *   acc[0..F)  += stats[i]/n              (KL_i batch mean; history['KL{i}'] = acc[i]/acc[F+3])
 *   acc[F]     += stats[F] + beta*sum_i stats[i]   (sample-weighted total loss; history['loss'] = acc[F]/acc[F+2])
 *   acc[F+1]   += stats[F+1]              (accuracy sum;  history['accuracy'] = acc[F+1]/acc[F+2])
 *   acc[F+2]   += n ;  acc[F+3] += 1      (samples, batches)
 * stats is the (all-reduced) vector written by dib_train_step / dib_forward; acc has F+4 floats. */
int dib_metrics_update(const float* stats, const float* beta_dev, float* acc, int32_t number_features, void* stream);
/* the same with the nonlinear IB term: acc[F] += stats[F] + n * beta * kl_loss_scale * (sum_i stats[i] / n)^kl_loss_exponent */
int dib_metrics_update_ex(const float* stats, const float* beta_dev, float* acc, int32_t number_features,
                          float kl_loss_exponent, float kl_loss_scale, void* stream);

/* utils.bhattacharyya_dist_mat (utils.py:177-212) followed by exp(-D) (visualization.py:34):
 * mu_logvar [n, 2E] -> out_dist [n, n] (may be NULL) and out_compression [n, n] (may be NULL). */
int dib_bhattacharyya(const float* mu_logvar, int64_t n, int32_t embedding_dimension,
                      float* out_dist, float* out_compression, void* stream);

/* NEXT ROW f2 -- pairwise closed forms between two sets of diagonal Gaussians, rows (mu || logvar):
 *   kind 0: utils.bhattacharyya_dist_mat(mus1, logvars1, mus2, logvars2)  (utils.py:177-212)
 *   kind 1: utils.kl_divergence_mat(mus1, logvars1, mus2, logvars2) = KL(N1_i || N2_j)  (utils.py:213-247)
 * mu_logvar_1 [n, 2E], mu_logvar_2 [m, 2E] -> out [n, m] and/or out_exp_neg [n, m] = exp(-out) (either may be NULL). */
int dib_pairwise_gaussian(int32_t kind, const float* mu_logvar_1, int64_t n, const float* mu_logvar_2, int64_t m,
                          int32_t embedding_dimension, float* out, float* out_exp_neg, void* stream);

/* NEXT ROW f2 -- visualization.save_compression_matrices (visualization.py:14-35) / SaveCompressionMatricesCallback
 * (models.py:152-186) / StashEmbeddingsCallback (nb-radial cell 5) for ALL features in one call: for feature i take
 * rows row_index[i, 0..n) of x [n_total, sum d_i] (row_index: device int32 [F, n], NULL = rows 0..n-1 for every
 * feature), run encoder i without noise, then Bhattacharyya and exp(-D).  Outputs (each may be NULL):
 * out_mu_logvar [F, n, 2E], out_dist [F, n, n], out_compression [F, n, n].  n <= config.max_batch. */
int dib_compression_matrices(dib_model* h, const float* params, const float* x, int64_t n_total,
                             const int32_t* row_index, int64_t n, float* out_mu_logvar, float* out_dist,
                             float* out_compression, void* workspace, void* stream);

/* NEXT ROW f3 -- utils.get_scaled_similarity (utils.py:127-175; distances utils.py:75-125):
 * kind 0 'l2sq' | 1 'l2' | 2 'l1' | 3 'linf' | 4 'cosine';  e1 [n, d], e2 [m, d] -> out [n, m] = similarity / temperature.
 * Every entry equals, bit for bit, the s_ij the streaming InfoNCE sweeps compute (dib_debug_infonce_stream in
 * dib_b200_test_hooks.h runs those). */
int dib_scaled_similarity(int32_t kind, const float* e1, int64_t n, const float* e2, int64_t m, int32_t d,
                          float temperature, float* out, void* stream);

/* NEXT ROW f3 -- the InfoNCE head of the custom training loop (train.py:203-213) and its reverse mode (train.py:216-219):
 *   S = get_scaled_similarity(e1, e2);  out_loss[0] = mean_i CE(i, S[i,:]) + mean_i CE(i, S^T[i,:])   (nats)
 *   d_e1, d_e2 [n, d] = d loss / d e1, d e2 (either may be NULL).  e1 = model(x) (feed d_e1 to dib_train_step of a
 *   DIB_LOSS_EXTERNAL model), e2 = the caller's output encoder.  scratch: n*n + 4n floats.  n <= 32768, d <= 512.
 *   'linf': the gradient of max_k |a_k - b_k| is split evenly between tied maximal coordinates, as TF's reduce_max does.
 *   tests/test_gpu_infonce_stream.py checks this head and the streaming sweeps (dib_debug_infonce_stream) element by
 *   element against float64 with per-element error bounds. */
int dib_infonce_head(int32_t kind, const float* e1, const float* e2, int64_t n, int32_t d, float temperature,
                     float* scratch, float* out_loss, float* d_e1, float* d_e2, void* stream);

/* NEXT ROW f1 -- utils.estimate_mi_sandwich_bounds' per-batch kernel (utils.py:36-65): InfoNCE lower and leave-one-out
 * upper bound (nats) of I(U;X) for one encoder on one batch of n samples.  mu_logvar [n, 2E] (dib_encode_feature
 * output); eps [n, E] or NULL -> Philox(seed, step, row, feature 0, dim); row_scratch [2n] floats; out [2]. */
int dib_mi_sandwich_bounds(const float* mu_logvar, int64_t n, int32_t embedding_dimension, const float* eps, uint64_t seed,
                           uint32_t step, float* row_scratch, float* out_lower_upper, void* stream);

/* NEXT ROW f1, batched -- the whole of utils.estimate_mi_sandwich_bounds / InfoPerFeatureCallback (models.py:188-223) in one
 * launch: `groups` = features x evaluation batches independent problems of n rows each, mu_logvar [groups, n, 2E] (the
 * out_mu_logvar of dib_compression_matrices with n = batches * batch size rows per feature is exactly this layout),
 * accumulated in float64 as the reference does (utils.py:40-41).  eps [groups, n, E] or NULL -> Philox keyed
 * ((seed << 8) + g / batches_per_feature; step g % batches_per_feature; row; feature 0; dim), i.e. the streams of the
 * per-feature, per-batch calls.  row_scratch: groups * n * 2 doubles; out: [groups, 2] doubles (lower, upper) in nats. */
int dib_mi_sandwich_bounds_batched(const float* mu_logvar, int32_t groups, int64_t n, int32_t embedding_dimension,
                                   const float* eps, uint64_t seed, int32_t batches_per_feature, double* row_scratch,
                                   double* out_lower_upper, void* stream);

/* nb-particle cell 8 (:521-570): per-probe InfoNCE lower / leave-one-out upper bounds (nats), float64, of m probe encodings
 * against `batches` batches of encoded data rows, in one launch of the main kernel.  probe_mu_logvar [m, 2E] and
 * data_mu_logvar [data_rows, 2E] are (mu || logvar) rows (dib_encode_feature output); batch b is rows
 * [batch_offsets[b], batch_offsets[b+1]) with batch_offsets a nondecreasing DEVICE int64 array of batches + 1 entries in
 * [0, data_rows], every batch at least one row.  For probe p and batch b, u = mu_p + exp(lv_p / 2) eps_pb and
 *   lower_pb = log p(u|x_p) - log( (p(u|x_p) + sum_j p(u|x_j)) / (N_b + 1) ),  upper_pb = log p(u|x_p) - log( sum_j p(u|x_j) / N_b )
 * evaluated in log space (finite where the linear-space upper bound underflows to log(x/0)); out [m, 2] = the means over b.
 * eps [batches, m, E] or NULL -> Philox keyed (seed, step b, row p, feature 0, dim), so a probe's result does not depend on
 * m.  scratch: dib_mi_bounds_at_probes_scratch_bytes(m, data_rows, batches, E), 256-byte aligned.  1 <= E <= 128,
 * 1 <= batches <= 65535, m < 2^31.  Deterministic: no atomics, repeated calls are bit-identical. */
int dib_mi_bounds_at_probes(const float* probe_mu_logvar, int64_t m, const float* data_mu_logvar,
                            const int64_t* batch_offsets, int32_t batches, int32_t embedding_dimension, const float* eps,
                            uint64_t seed, void* scratch, double* out_lower_upper, void* stream);
size_t dib_mi_bounds_at_probes_scratch_bytes(int64_t m, int64_t data_rows, int32_t batches, int32_t embedding_dimension);

/* NEXT ROW f4 -- ctw.estimate_entropy(seq, alphabet_size) (chaos/ctw.pyx:2-3 -> chaos/cppctw.cpp:163-171): infinite-depth
 * Context-Tree-Weighting entropy-rate estimate in bits/symbol.  HOST functions on HOST memory (the suffix-tree build is
 * irregular pointer chasing; SURVEY 8f keeps it on the CPU): symbols are int8 in [0, alphabet_size), alphabet_size <= 127.
 * The batch form runs `count` independent sequences (sequences + offsets[i] .. offsets[i+1]) on num_threads host threads
 * (<= 0: all cores).  Results are bit-identical to the reference (double carrying a float-rounded value). */
int dib_ctw_estimate_entropy(const int8_t* sequence, int64_t length, int32_t alphabet_size, double* out_bits_per_symbol);
int dib_ctw_estimate_entropy_batch(const int8_t* sequences, const int64_t* offsets, int32_t count, int32_t alphabet_size,
                                   int32_t num_threads, double* out_bits_per_symbol);
const char* dib_ctw_last_error(void);

/* ---- observability (no reference counterpart) ---------------------------------------------------------
 * dib_launch_count: kernels launched by this library in this process.
 * dib_profile_enable(h,1): bracket every launch group of subsequent forward/train_step calls with CUDA events
 * recorded on the caller's stream; dib_profile_read waits for them and returns up to `capacity` durations (ms)
 * with '\n'-separated labels; dib_profile_enable(h,0) turns it off and frees the events. */
uint64_t dib_launch_count(void);
int dib_profile_enable(dib_model* h, int32_t on);
int32_t dib_profile_read(dib_model* h, char* labels, size_t labels_bytes, float* ms, int32_t capacity);

/* bring-up switch for THIS handle (bit mask, 0 = the default kernels): 1 = unfused encoder kernels, 2 = integration network on
 * fp32-storage TF32 kernels, 4 = no fused integration tail (per-layer 16-bit GEMMs plus a head kernel), 8 = the generic head
 * kernel even when output_dimensionality == 1, 16 = the fused tail without its dgrad stages (the backward launches those
 * dgrads separately).  dib_model_info reports the resulting path. */
int dib_debug_force_unfused(dib_model* h, int32_t on);

/* text of the last error raised on this thread ("" if none). */
const char* dib_last_error(void);

/* "sm_90a" etc: the architecture the kernels were compiled for, and the ABI version. */
const char* dib_build_info(void);

/* one line describing what THIS handle runs, e.g.
 * "precision=fp16 encoders=fused-wgmma-f16 integration=int16-wgmma-f16 operands=fp16 accumulate=fp32".  The 16-bit path adds
 * its tail ("integration_tail=fwd2-head-dgrad" / "fwd2-head") or, without a fused tail, its head kernel
 * ("integration_head=head1" / "generic").
 * Returns the number of bytes written (excluding the terminator), negative on error. */
int32_t dib_model_info(const dib_model* h, char* out, size_t out_bytes);

#ifdef __cplusplus
}
#endif
#endif /* DIB_B200_H_ */
