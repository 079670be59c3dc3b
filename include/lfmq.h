/* lfmq.h -- C ABI of the GPU-native (H100, sm_90a) training / inference step for the lfm_quant recurrent
 * forecaster (RNNPointEstimate, LSTM cell, forecast_steps = 1).
 *
 * The reference (lakshaykc/lfm_quant) defines no FFI: its seam is the Python protocol between the
 * drivers (scripts/train.py, scripts/predict.py) and the Keras model / Dataset objects.  Each entry
 * point below names the reference call site(s) it replaces (paths relative to /root/reference/scripts).
 * The Python mirror of that protocol lives in lfm_quant_b200/ and reaches this library via ctypes;
 * INTEGRATION.md shows the binding a reference maintainer would add.
 *
 * Conventions
 *   - plain C types only; every device pointer is caller-owned (the Python host allocates with torch and
 *     passes tensor.data_ptr()); the library never allocates device memory.
 *   - all tensors are dense row-major fp32 unless stated; x is [B, T, F], y/preds are [B, T, O].
 *   - every call that touches the device takes a cudaStream_t (as void*) and is asynchronous.
 *   - return value: 0 on success, else an LFMQ_ERR_* code; lfmq_last_error() gives the message
 *     (thread-local).  A handle is not thread-safe; different handles may run at the same time from different host
 *     threads on different streams, each with a device share (lfmq_set_device_share) when they share a GPU.
 */
#ifndef LFMQ_H_
#define LFMQ_H_

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define LFMQ_ABI_VERSION 4   /* 3: LFMQ_PREC_BF16X3, general tensor-core path; 4: lfmq_chain_* (forecast_steps > 1), lfmq_window_index */

enum { LFMQ_OK = 0, LFMQ_ERR_ARG = 1, LFMQ_ERR_CUDA = 2, LFMQ_ERR_UNSUPPORTED = 3, LFMQ_ERR_WORKSPACE = 4 };
enum { LFMQ_OPT_ADADELTA = 0, LFMQ_OPT_ADAM = 1, LFMQ_OPT_RMSPROP = 2, LFMQ_OPT_SGD = 3 };
/* LFMQ_PREC_FP32:   fp32 SIMT arithmetic everywhere (the parity mode, <=1e-4 rel vs the oracle; any cell / head).
 * LFMQ_PREC_BF16:   gate GEMMs on wgmma tensor cores with bf16 operands, fp32 accumulate, fp32 cell state.
 *                   num_hidden a multiple of 64 (<= 512), any num_layers, dropout and recurrent dropout.  Training: LSTM
 *                   cell, point-estimate head.  forward_only handles: LSTM or GRU cell, point-estimate or uq head (uq:
 *                   Dropout / recurrent dropout stay active, as on the fp32 path).  The LSTM point estimate at H = 256 /
 *                   L = 1 without recurrent dropout runs the persistent cluster kernels.
 * LFMQ_PREC_BF16X3: fp32-tolerance forward on tensor cores (forward_only handles: predict.py:129), same cells and heads
 *                   as forward_only LFMQ_PREC_BF16: every operand split into bf16 high + low halves, three wgmma products
 *                   per GEMM (hi*hi + lo*hi + hi*lo), accurate expf / tanhf gate nonlinearities, fp32 head -- <=1e-4 rel
 *                   vs the oracle.
 * LFMQ_PREC_TF32:   the LFMQ_PREC_FP32 step with its GEMMs on wgmma tensor cores: operands rounded to tf32 (cvt.rna:
 *                   nearest, ties away from zero), fp32 accumulation.  Pointwise cell algebra, carried state, BN /
 *                   dropout, heads' activations, losses, clip, optimizer and MaxNorm are the fp32 path's own.  Any cell,
 *                   head, num_layers and chain, trainable or forward_only, and the same parameter layout as fp32 (a
 *                   checkpoint moves freely between precisions).  Deterministic like fp32: a row's outputs do not depend
 *                   on the other rows or the launch size, and two backward calls give the same bits.  Dense handles
 *                   refuse it. */
enum { LFMQ_PREC_FP32 = 0, LFMQ_PREC_BF16 = 1, LFMQ_PREC_BF16X3 = 2, LFMQ_PREC_TF32 = 3 };

/* config.rnn_cell (lfm_quant.py:39; rnn_point_estimate.py:80-102).  GRU is Keras' default reset_after=True cell:
 * 3 gate blocks z|r|h, bias [2][3H] (input row, recurrent row).  The tensor-core precisions train the LSTM cell only;
 * they run the GRU cell on forward_only handles. */
enum { LFMQ_CELL_LSTM = 0, LFMQ_CELL_GRU = 1 };

typedef struct lfmq_handle_s* lfmq_handle;

/* Static description of one model instance.  Field names follow the reference's flags
 * (lfm_quant.py:23-106) and Dataset attributes (data_processing.py:37,82-88). */
typedef struct lfmq_config {
  int32_t struct_size;       /* sizeof(lfmq_config), ABI guard */
  int32_t max_batch;         /* largest B any call will pass (per rank) */
  int32_t seq_len;           /* T = max_unrollings          (data_processing.py:37) */
  int32_t n_inputs;          /* F = n_fin + n_aux           (data_processing.py:82) */
  int32_t n_outputs;         /* O = n_fin                   (data_processing.py:83) */
  int32_t num_hidden;        /* H                            (lfm_quant.py:53) */
  int32_t num_layers;        /* L                            (lfm_quant.py:51) */
  int32_t target_idx;        /* Dataset.target_index         (data_processing.py:88) */
  int32_t train;             /* config.train: Dropout / recurrent dropout active (rnn_point_estimate.py:87,89) */
  int32_t precision;         /* LFMQ_PREC_* */
  int32_t optimizer;         /* LFMQ_OPT_*                   (optimizers.py:21-27) */
  int32_t forward_only;      /* 1: no backward workspace (predict.py) */
  int32_t rnn_cell;          /* LFMQ_CELL_*: config.rnn_cell 'lstm' | 'gru' (rnn_point_estimate.py:80,90) */
  int32_t uq;                /* config.UQ: 0 = RNNPointEstimate, 1 = RNNUqRangeEstimate (model_utils/model.py:25-33):
                              * target + variance heads, Gaussian-NLL loss, dropout always active
                              * (rnn_uq_range_estimate.py:86,88,104-108).  fp32 path, single GPU. */
  float dropout;             /* lfm_quant.py:61 */
  float recurrent_dropout;   /* lfm_quant.py:62 */
  float target_lambda;       /* lfm_quant.py:69 */
  float rnn_lambda;          /* lfm_quant.py:70 */
  float max_grad_norm;       /* lfm_quant.py:55; <= 0 disables clipping (train.py:195) */
  float max_norm;            /* MaxNorm on each LSTM kernel (rnn_point_estimate.py:85) */
  float sgd_momentum;        /* lfm_quant.py:93 */
  float bn_epsilon;          /* keras BatchNormalization default 1e-3 */
  uint64_t seed;             /* keys the Philox dropout streams */
} lfmq_config;

/* Thread-local message for the last non-zero return code. */
const char* lfmq_last_error(void);
int32_t lfmq_abi_version(void);

/* Bytes of device workspace lfmq_create needs for this config (parameters, gradients, optimizer
 * slots, saved activations).  The caller allocates it (torch.empty(..., dtype=uint8, device='cuda')). */
int32_t lfmq_workspace_bytes(const lfmq_config* cfg, uint64_t* bytes);

/* Replaces Model(config, dataset).get_model() (model_utils/model.py:20-39) and
 * RNNPointEstimate.__init__/_build_model (models/point_estimate/rnn_point_estimate.py:24-107).
 * Parameters start zeroed except BN moving_variance = 1; the host initialiser
 * (model_utils/initializers.py:14-24) uploads weights with lfmq_set_params. */
int32_t lfmq_create(const lfmq_config* cfg, void* workspace, uint64_t workspace_bytes, lfmq_handle* out);
int32_t lfmq_destroy(lfmq_handle h);

/* Handles that run concurrently on one GPU (ensembles: runtime/model_execution.py:154-199 trains and predicts N members).
 * Some launches of the general tensor-core path are persistent: their CTAs wait for each other at a barrier in global
 * memory, which needs all of them resident at once.  lfmq_set_device_share(h, num, den) lets such a launch of h count on
 * num/den of the SMs only (fewer CTAs than that budget, else the steps are launched one by one).  Default 1/1, the whole
 * device.  Give every handle that may run at the same time as others on the same GPU a share, with the shares summing
 * to at most 1; launches that do not wait across CTAs need none.  Host-only; takes effect from the next call. */
int32_t lfmq_set_device_share(lfmq_handle h, int32_t num, int32_t den);
/* The CTA budget of one persistent launch under a share (host arithmetic, no device): sm_count * ctas_per_sm for the
 * whole device, else floor(sm_count * num / den), one CTA per SM. */
int32_t lfmq_persistent_cta_budget(int32_t sm_count, int32_t ctas_per_sm, int32_t num, int32_t den, int64_t* budget);

/* ---- the linear baseline: MLPLinearPointEstimate (models/point_estimate/mlp_linear_point_estimate.py:66-77) ----
 * One Dense(O) layer OUTPUT_1 over the flattened input window: preds[B,O] = x[B, T*F] W[T*F, O] + b.  x is the [B,T,F]
 * batch viewed as [B, T*F] (data_processing.py:363-365); y and preds are the last step only, [B,O].  A dense handle is
 * an ordinary lfmq_handle: lfmq_param_count / lfmq_param_spec (OUTPUT_1/kernel [T*F, O], OUTPUT_1/bias [O]), the
 * parameter, gradient and optimizer-slot pointers, lfmq_set_params / lfmq_get_params, lfmq_apply (clip and optimizer;
 * no MaxNorm), lfmq_set_device_share, profiling and lfmq_destroy work on it unchanged, and
 *   lfmq_forward     x [B, T*F] -> preds [B,O] (step and row0 are ignored: the model has no dropout)
 *   lfmq_loss        the MLP branch of Losses._get_loss_point_estimate (losses.py:69-75,100-115) in its MSE form, as
 *                    validation evaluates it (is_validation=True): out_dev = {target_lambda * mse_0 +
 *                    (1 - target_lambda) * mse_all, mse_0}; rows whose targets are all zero have their predictions
 *                    zeroed and count in both denominators, B and B * O
 *   lfmq_mask_count  out_dev = {B, rows whose targets are not all zero}, as on a recurrent handle
 *   lfmq_backward    forward, the loss (Keras Huber terms when huber_loss, losses.py:102-105) and the gradients of the
 *                    kernel and the bias; denom_dev = {B_global, ...} (lfmq_mask_count summed over the ranks) or NULL
 *   lfmq_train_step  lfmq_backward + lfmq_apply, loss_out_dev = {loss, mse_0}
 * dispatch on it.  The uq and chain entry points refuse it.  fp32 only: the model reads every byte of x once for O
 * multiply-adds each, so it is bound by memory, not arithmetic, and LFMQ_PREC_BF16 / LFMQ_PREC_BF16X3 are refused at
 * create with LFMQ_ERR_UNSUPPORTED.  All kernels are deterministic (fixed reduction orders, no atomics); a row's
 * prediction does not depend on the other rows of the batch. */
typedef struct lfmq_dense_config {   /* 56 bytes: 10 int32 + 4 float */
  int32_t struct_size;       /* sizeof(lfmq_dense_config), ABI guard */
  int32_t max_batch;         /* largest B any call will pass (per rank) */
  int32_t seq_len;           /* T */
  int32_t n_inputs;          /* F; the kernel has T * F rows (<= 48 * 1024) */
  int32_t n_outputs;         /* O */
  int32_t target_idx;        /* Dataset.target_index */
  int32_t precision;         /* LFMQ_PREC_FP32 */
  int32_t optimizer;         /* LFMQ_OPT_* */
  int32_t forward_only;      /* 1: no gradient or optimizer workspace (predict.py) */
  int32_t huber_loss;        /* config.huber_loss: the training loss uses Keras Huber terms (losses.py:102-105) */
  float target_lambda;       /* lfm_quant.py:69 */
  float huber_delta;         /* config.huber_delta */
  float max_grad_norm;       /* <= 0 disables clipping (train.py:195) */
  float sgd_momentum;
} lfmq_dense_config;
int32_t lfmq_dense_workspace_bytes(const lfmq_dense_config* cfg, uint64_t* bytes);
/* Replaces MLPLinearPointEstimate(config, dataset).model.  Parameters start zeroed; the host initialiser uploads them
 * with lfmq_set_params. */
int32_t lfmq_dense_create(const lfmq_dense_config* cfg, void* workspace, uint64_t workspace_bytes, lfmq_handle* out);

/* model.trainable_variables / model.weights (train.py:192,198): tensors are listed in Keras order,
 * trainable ones first: per layer lstm_l/{kernel,recurrent_kernel,bias} (gru_l/... with bias [2][3H] for LFMQ_CELL_GRU), batch_normalization[_k]/{gamma,beta};
 * OUTPUT_1/{kernel,bias} (uq: OUTPUT_TARGET_1/{kernel,bias}, OUTPUT_VARIANCE_1/{kernel,bias}); then per layer batch_normalization[_k]/{moving_mean,moving_variance}. */
int32_t lfmq_param_count(lfmq_handle h, int32_t* n_tensors, int64_t* n_trainable_elems, int64_t* n_total_elems);
int32_t lfmq_param_spec(lfmq_handle h, int32_t index, char* name, int32_t name_cap, int32_t* ndim,
                        int64_t shape[2], int64_t* offset_elems, int32_t* trainable);
/* Device pointers into the workspace: flat fp32 parameters [n_total]; flat gradients
 * [n_trainable + LFMQ_TAIL_LEN] whose tail holds {loss, mse_0} contributions of the last lfmq_backward,
 * {grad_norm, clip_scale} of the last lfmq_apply and, on a uq handle, uq_loss_last_tar (the loss slot is then the
 * weighted uq loss); optimizer slots [n_slots * n_trainable]. */
enum { LFMQ_TAIL_LOSS = 0, LFMQ_TAIL_MSE0 = 1, LFMQ_TAIL_GRAD_NORM = 2, LFMQ_TAIL_CLIP_SCALE = 3,
       LFMQ_TAIL_UQ_LOSS_LAST_TAR = 4, LFMQ_TAIL_LEN = 8 };   /* grads[n_trainable + LFMQ_TAIL_*] */
/* Row weights of the training loss (DESIGN.md section 6d).  w_dev: a device vector of at least max_batch floats, each
 * >= 0 and finite, or NULL (the default) for the unweighted step.  Row b of each later call's batch weighs w_dev[b]: b is
 * the shard's own row, and row0 does not shift it.  The pointer is kept, not copied: write the next batch's weights
 * into it on the handle's stream.  Every mean of the training loss becomes a weighted mean (the all-zero-target mask
 * still multiplies in), so the tail's loss entries are the weighted loss; weights of 1 give the same bits as NULL.
 * Read by lfmq_backward, lfmq_train_step, lfmq_mask_count, lfmq_mask_count_uq (their counts become {sum of weights,
 * weighted unmasked rows[, weighted unmasked last-step rows]}, which data parallelism all-reduces as before; with
 * weights, lfmq_mask_count forms the counts in the handle's own scalar block and copies the first two to out_dev),
 * lfmq_chain_backward(_dp) and lfmq_chain_mask_count, where each stage reads its own handle's pointer.  No *_loss*
 * entry point reads it: validation stays unweighted.  A batch whose weights sum to 0 has loss 0 and gradient 0 (a
 * weighted count of 0 divides as 1).  Recurrent and dense handles; forward_only handles get LFMQ_ERR_UNSUPPORTED. */
int32_t lfmq_set_row_weights(lfmq_handle h, const float* w_dev);
int32_t lfmq_params_ptr(lfmq_handle h, float** dev);
int32_t lfmq_grads_ptr(lfmq_handle h, float** dev);
int32_t lfmq_opt_state_ptr(lfmq_handle h, float** dev, int64_t* n_elems);
/* model.load_weights / save_weights payload (train.py:87,99,171; predict.py:93): host <-> device copy
 * of the flat parameter vector. */
int32_t lfmq_set_params(lfmq_handle h, const float* host, int64_t n_elems, void* stream);
int32_t lfmq_get_params(lfmq_handle h, float* host, int64_t n_elems, void* stream);

/* model(inp) / model.predict(inp) (train.py:182,289; predict.py:129): preds[B,T,O] = Dense(Dropout(BN(LSTM(x)))).
 * Dropout is active iff cfg.train (rnn_point_estimate.py:87,89); `step` and `row0` (global index of
 * the first row of this shard) key the dropout streams so masks are independent of the GPU count. */
int32_t lfmq_forward(lfmq_handle h, const float* x, int32_t B, int64_t row0, int64_t step, float* preds, void* stream);
/* model(inp) / model.predict(inp) of RNNUqRangeEstimate (train.py:204-206, predict.py:135-138): preds[0] -> preds,
 * preds[1] -> var, both [B,T,O].  Dropout masks are drawn for (step, row0) on every call, also with train = 0
 * (rnn_uq_range_estimate.py:86,88 pass training=True literally).  uq handles only; lfmq_forward refuses them. */
int32_t lfmq_forward_uq(lfmq_handle h, const float* x, int32_t B, int64_t row0, int64_t step, float* preds, float* var,
                        void* stream);

/* Losses.weight_adjusted_mse([y],[pred]) (model_utils/losses.py:19-135), RNN branch, forecast_steps=1.
 * out_dev[0] = loss, out_dev[1] = mse_0 (device floats).  Used for validation (train.py:329). */
int32_t lfmq_loss(lfmq_handle h, const float* preds, const float* y, int32_t B, float* out_dev, void* stream);
/* Losses.weight_adjusted_uq_loss([y],[pred],[var]) (model_utils/losses.py:137-284), RNN branch, forecast_steps=1.
 * out_dev = {uq_loss, uq_loss_last_tar, mse_0}.  A zero-padded step makes uq_loss NaN, as the reference's formula does. */
int32_t lfmq_loss_uq(lfmq_handle h, const float* preds, const float* var, const float* y, int32_t B, float* out_dev,
                     void* stream);

/* Number of unmasked [b,t] rows of y (losses.py:72-73,132): out_dev[0] = B, out_dev[1] = sum(mask).
 * Under data parallelism the host all-reduces these two floats once per batch and passes the result
 * as `denom_dev` below. */
int32_t lfmq_mask_count(lfmq_handle h, const float* y, int32_t B, float* out_dev, void* stream);
/* The counts behind the uq loss (losses.py:179-284): out_dev = {B, sum(mask), sum(mask[:, T-1])}, the denominators of
 * mse_0, of the mean over the mask and of the means over the last step.  Under data parallelism the host all-reduces
 * these three floats once per batch and passes the result as `denom_dev` of lfmq_backward on a uq handle. */
int32_t lfmq_mask_count_uq(lfmq_handle h, const float* y, int32_t B, float* out_dev, void* stream);

/* First half of Train._train_step_point (train.py:181-192): forward, loss, BPTT.  Fills the flat
 * gradient buffer (+ its 4-float tail).  denom_dev = device {B_global, mask_count_global} or NULL to use
 * this call's own batch.  With N ranks the host all-reduces grads[0 : n_trainable+2] (SUM) next.
 * On a uq handle (train.py:201-218) denom_dev = the three counts of lfmq_mask_count_uq summed over the ranks; the tail
 * entries {uq_loss, mse_0, uq_loss_last_tar} are then this shard's contributions, and the host reduces the gradient
 * and them through lfmq_chain_grad_pack / lfmq_chain_grad_unpack with n_stages = 1.
 * Stream semantics: everything is ordered on `stream`. */
int32_t lfmq_backward(lfmq_handle h, const float* x, const float* y, int32_t B, int64_t row0, int64_t step,
                      const float* denom_dev, void* stream);

/* Second half (train.py:195-198 + the MaxNorm kernel constraint): clip_by_global_norm over the flat
 * gradient, optimizer update with learning rate `lr` (host-evaluated schedule, optimizers.py:31-54),
 * `iteration` = optimizer.iterations before this update. */
int32_t lfmq_apply(lfmq_handle h, float lr, int64_t iteration, void* stream);

/* Whole step for one GPU: lfmq_backward + lfmq_apply.  loss_out_dev (may be NULL) receives {loss, mse_0}; on a uq
 * handle {uq_loss_last_tar, mse_0}, the pair Train._train_step_uq_range returns (train.py:225). */
int32_t lfmq_train_step(lfmq_handle h, const float* x, const float* y, int32_t B, int64_t row0, int64_t step,
                        float lr, float* loss_out_dev, void* stream);

/* ---- forecast_steps > 1 (models/point_estimate/rnn_point_estimate.py:109-150; models/model_base_class.py:18-51) ----
 * The Keras graph of S forecast steps is S stages: stage 0 = the trunk handle (num_layers layers + OUTPUT_1); stage
 * s >= 1 = one more handle with num_layers = 1 (lstm_{L+s} / gru_{L+s}, its BatchNormalization and Dropout, OUTPUT_{s+1})
 * created with the same seq_len / n_inputs / n_outputs / max_batch.  Stage s reads the previous stage's input window
 * shifted by one step with [pred_{s-1}[:, T-1, :], aux features of the last ORIGINAL step] appended (:113-124).
 * `stages`, `preds`, `y` are host arrays of n_stages (<= 8) entries; `weights` = config.forecast_steps_weights (host).
 * `work`: device floats, n_stages * B * seq_len * n_inputs (stage inputs + one input-gradient buffer).
 * Dropout streams of stage s continue the trunk's layer numbering (layer num_layers + s - 1).
 * Training-mode stages (cfg.train) run on the LFMQ_PREC_FP32 or LFMQ_PREC_TF32 kernels; forward_only stages may use any
 * precision.
 * Every stage of one chain has the same cfg.uq.  A uq chain (models/uq_range_estimate/rnn_uq_range_estimate.py:114-157)
 * gives every stage the heads OUTPUT_TARGET_{s+1} and OUTPUT_VARIANCE_{s+1}, keeps Dropout / recurrent dropout on in
 * every stage and builds each next window from the previous stage's TARGET predictions (variances never feed forward).
 * It runs lfmq_chain_forward_uq and lfmq_chain_loss_uq; lfmq_chain_backward and lfmq_chain_apply serve both kinds. */
/* model(inp) -> [pred_1 .. pred_S], each [B,T,O] (train.py:182, predict.py:129) */
int32_t lfmq_chain_forward(const lfmq_handle* stages, int32_t n_stages, const float* x, int32_t B, int64_t row0,
                           int64_t step, float* const* preds, float* work, void* stream);
/* Losses.weight_adjusted_mse(y_true list, y_pred list) (losses.py:19-53): out_dev = {sum_s w_s loss_s, sum_s w_s mse_s} */
int32_t lfmq_chain_loss(const lfmq_handle* stages, int32_t n_stages, const float* const* preds, const float* const* y,
                        const float* weights, int32_t B, float* out_dev, void* stream);
/* uq chain: model(inp) -> [tar_1, var_1, .., tar_S, var_S] (train.py:204-206, predict.py:135-138): preds[s] and vars[s],
 * each [B,T,O], Dropout masks drawn for (step, row0) on every call */
int32_t lfmq_chain_forward_uq(const lfmq_handle* stages, int32_t n_stages, const float* x, int32_t B, int64_t row0,
                              int64_t step, float* const* preds, float* const* vars, float* work, void* stream);

/* ---- Monte-Carlo dropout samples of a uq model in one prediction --------------------------------------------------
 * The reference's UQ inference (runtime/model_execution.py:201-241, utils/post_processing.py:39-75) runs one dropout
 * sample per process and combines the members' files.  These entry points draw `samples` >= 1 samples of every window
 * in one call: sample s of window b is global row row0 + s * B + b of the batch tiled `samples` times, with that row's
 * dropout masks.  Sample 0 is therefore lfmq_forward_uq / lfmq_chain_forward_uq at (step, row0), and the samples are
 * independent draws.  The samples * B rows run in launches of at most max_batch rows (the smallest of the stages'), so
 * B and samples are not bounded by max_batch; a chain runs each replica's own trajectory.  After each launch one pass
 * folds its samples, in increasing s, into four [B,T,O] fp32 arrays per stage (Welford, fixed order, no atomics):
 *   mean_pred, mean_var   the sample means of the target predictions and of the predicted variances
 *   var_pred, var_var     their population variances (divided by samples)
 * The results do not depend on how the rows are cut into launches, nor on the other windows of the batch.  Point-estimate
 * and dense handles are refused with LFMQ_ERR_ARG (their dropout is off at prediction time).  `work`: caller-owned device
 * scratch, 256-byte aligned, of the size the matching *_work_bytes query gives for (B, samples). */
int32_t lfmq_forward_uq_mc_work_bytes(lfmq_handle h, int32_t B, int32_t samples, uint64_t* bytes);
int32_t lfmq_forward_uq_mc(lfmq_handle h, const float* x, int32_t B, int64_t row0, int64_t step, int32_t samples,
                           float* mean_pred, float* mean_var, float* var_pred, float* var_var, void* work,
                           uint64_t work_bytes, void* stream);
/* The same for a uq chain (stages as lfmq_chain_forward_uq); the four outputs are host arrays of n_stages pointers. */
int32_t lfmq_chain_forward_uq_mc_work_bytes(const lfmq_handle* stages, int32_t n_stages, int32_t B, int32_t samples,
                                            uint64_t* bytes);
int32_t lfmq_chain_forward_uq_mc(const lfmq_handle* stages, int32_t n_stages, const float* x, int32_t B, int64_t row0,
                                 int64_t step, int32_t samples, float* const* mean_pred, float* const* mean_var,
                                 float* const* var_pred, float* const* var_var, void* work, uint64_t work_bytes,
                                 void* stream);
/* ---- predictive quantiles and proper scores of those samples ------------------------------------------------------
 * The samples of lfmq_chain_forward_uq_mc, and with them its four moment arrays, bit for bit (the same launches and
 * the same fold).  Each launch's samples at [T-1, target_idx] are also gathered into `work` as mu[s][b][m] and
 * v[s][b][m], and after the last launch one pass treats each (window, stage) as the Gaussian mixture
 * F(q) = (1/M) sum_m Phi((q - mu_m) / sigma_m), sigma_m^2 = v_m, M = samples, and writes (device fp32):
 *   quantiles[s] [B][n_levels]  the q with F(q) = levels[k]: bracketed by the smallest and largest component quantile
 *                               mu_m + sigma_m Phi^-1(levels[k]), refined by safeguarded Newton steps on the smaller
 *                               tail (1 - F(q) = 1 - level above the median) until |F(q) - level| <= 1e-6
 *                               min(level, 1 - level), the bracket is narrower than 1e-6 min_m sigma_m, or 64 steps;
 *   scores[s] [B][3]            with y (host array of n_stages device pointers, laid out as lfmq_chain_loss_uq takes
 *                               the targets) and the target y[s][b, T-1, target_idx]: {crps, nll, pit} =
 *                               {E|X - y| - E|X - X'| / 2 in the closed form for Gaussian mixtures (Grimit et al.
 *                               2006) over the M components and the M (M + 1) / 2 pairs, -log f(y) by log-sum-exp,
 *                               F(y)}.  A NaN target gives NaN scores (its quantiles are still written).  y == NULL:
 *                               scores is not written and may be NULL.
 * Every lane evaluates components in fp32 (the log-score terms in fp64) and sums in fp64; a warp adds its lanes in a
 * fixed tree, without atomics, so a window's outputs depend neither on the other windows nor on max_batch or where
 * launches are cut, and two calls give the same bits.  Accepted: uq chains as lfmq_chain_forward_uq_mc, any precision.
 * Point-estimate and dense handles, n_levels outside [1, 32], levels not strictly increasing inside (0, 1) (host float
 * [n_levels]) and null pointers: LFMQ_ERR_ARG.  The handles' parameters, gradients and optimizer slots are left
 * untouched.  `work`: caller-owned device scratch, 256-byte aligned, of the size the *_work_bytes query gives: that of
 * lfmq_chain_forward_uq_mc, then mu and v of every stage (2 * n_stages * B * samples floats). */
int32_t lfmq_chain_forward_uq_dist_work_bytes(const lfmq_handle* stages, int32_t n_stages, int32_t B, int32_t samples,
                                              int32_t n_levels, uint64_t* bytes);
int32_t lfmq_chain_forward_uq_dist(const lfmq_handle* stages, int32_t n_stages, const float* x, const float* const* y,
                                   int32_t B, int64_t row0, int64_t step, int32_t samples, const float* levels,
                                   int32_t n_levels, float* const* mean_pred, float* const* mean_var,
                                   float* const* var_pred, float* const* var_var, float* const* quantiles,
                                   float* const* scores, void* work, uint64_t work_bytes, void* stream);
/* ---- integrated gradients of the point forecast ---------------------------------------------------------------------
 * Which input fields and quarters of each window drive its forecast f(x) = pred[b, T-1, target_idx] (predict.py's
 * norm_preds_1), with dropout off and BatchNormalization in its inference form.  With the baseline x' = 0 (the value
 * the batcher pads with) and `steps` = M >= 1 midpoint-rule interpolants alpha_k = (k + 1/2) / M:
 *   attr[b,t,f] = x[b,t,f] * (1/M) sum_{k<M} df/dx[t,f] (alpha_k x[b])        attr [B,T,F]
 *   f_x[b] = f(x[b]), f_base[b] = f(0)                                           f_x, f_base [B]
 * so that sum_{t,f} attr[b] = f_x[b] - f_base[b] up to the quadrature error (completeness).  Interpolant k of window b
 * is row k * B + b of the batch tiled M times; those rows run in launches of at most max_batch rows, each one forward,
 * a one-hot seed of d pred at [T-1, target_idx], and the backward of the dz / dh chain and the dx GEMMs only (no
 * parameter gradient is formed).  One pass per launch adds its input gradients into attr in increasing k (fixed order,
 * no atomics).  A window's outputs do not depend on the other windows, their order, max_batch or where launches are
 * cut; two calls give the same bits; f_x and f_base are lfmq_forward's target column at x and at 0 bit for bit.  The
 * handle's parameters, gradient buffer (tail included) and optimizer slots are left untouched: a model may be
 * attributed between train steps.  B and steps are not bounded by max_batch.
 * Accepted: point-estimate handles with forward_only = 0 and train = 0, precision LFMQ_PREC_FP32 or LFMQ_PREC_TF32, either
 * cell, any num_layers.  LFMQ_PREC_BF16 / LFMQ_PREC_BF16X3 handles: LFMQ_ERR_UNSUPPORTED (their backward does not form
 * the lowest layer's input gradient).  forward_only, train = 1, uq and dense handles: LFMQ_ERR_ARG.
 * `work`: caller-owned device scratch, 256-byte aligned, of the size the *_work_bytes query gives for (B, steps). */
int32_t lfmq_integrated_gradients_work_bytes(lfmq_handle h, int32_t B, int32_t steps, uint64_t* bytes);
int32_t lfmq_integrated_gradients(lfmq_handle h, const float* x, int32_t B, int32_t steps, float* attr, float* f_x,
                                  float* f_base, void* work, uint64_t work_bytes, void* stream);
/* ---- permutation importance -----------------------------------------------------------------------------------------
 * How much the held-out loss depends on each group of input columns (Breiman 2001; Fisher, Rudin & Dominici 2019).
 * x [N,T,F] (or [N,T*F] on a dense handle) are the model's inputs, y[s] its targets; column c = t * F + f of a window
 * belongs to group col_group[c] in [0, G) (host int32 [T*F]).  Copy (g, r), for g < G and r < repeats, is the held-out
 * set with group g's columns taken from window pi(i) of the bijection pi = pi_{seed,g,r} of [0, N)
 * (lfmq_permutation_index); the targets stay.  Each copy runs in launches of at most max_batch rows keyed by the window
 * index (row0 = the launch's first window), so window i draws the same dropout masks at `step` in every copy.  Its
 * predictions fill a copy-sized buffer in `work`, which the loss entry point of the model then reduces: lfmq_loss (one
 * point or dense stage), lfmq_chain_loss with `weights` (host float [n_stages], the forecast-step weights), lfmq_loss_uq
 * or lfmq_chain_loss_uq.  out_dev [1 + G * repeats][3] (device): row 0 the unpermuted set, row 1 + g * repeats + r copy
 * (g, r); {loss, mse_0, 0} on point and dense stages, {uq_loss, uq_loss_last_tar, mse} on uq stages.
 * Accepted: S >= 1 point or uq stages of one chain (any precision, forward_only or not), or one dense handle.  The
 * handles' parameters, gradient buffers (tail included) and optimizer slots are left untouched.  repeats, N or G < 1, a
 * col_group value outside [0, G) or a null pointer: LFMQ_ERR_ARG.  `work`: caller-owned device scratch, 256-byte
 * aligned, of the size the *_work_bytes query gives for N: one launch's rows (per stage), the col_group copy and one
 * copy's predictions (and variances). */
int32_t lfmq_chain_permutation_importance_work_bytes(const lfmq_handle* stages, int32_t n_stages, int32_t N,
                                                     uint64_t* bytes);
int32_t lfmq_chain_permutation_importance(const lfmq_handle* stages, int32_t n_stages, const float* x,
                                          const float* const* y, const float* weights, int32_t N,
                                          const int32_t* col_group, int32_t G, int32_t repeats, uint64_t seed,
                                          int64_t step, float* out_dev, void* work, uint64_t work_bytes, void* stream);
/* The bijection of lfmq_chain_permutation_importance (host arithmetic, no device): *out = pi_{seed,group,repeat}(i).
 * m is the smallest even integer >= 2 with 2^m >= N and h = m / 2.  A 4-round Feistel network on [0, 2^m) splits
 * v = (L << h) | R; round j in 0..3 sets (L, R) <- (R, L ^ (philox4x32_10(R, j, group, repeat; seed_lo, seed_hi)[0] &
 * (2^h - 1))).  Starting from v = i, the network is applied until v < N (cycle walking). */
int32_t lfmq_permutation_index(int32_t N, uint64_t seed, int32_t group, int32_t repeat, int32_t i, int32_t* out);
/* ---- Shapley attributions ------------------------------------------------------------------------------------------
 * Which groups of input columns move each window's forecast, by permutation-sampling Shapley values (Strumbelj &
 * Kononenko 2014) with antithetic orderings (Mitchell et al. 2022).  x [N,T,F] (or [N,T*F] on a dense handle) are the
 * model's inputs; column c = t * F + f belongs to group col_group[c] in [0, G) (host int32 [T*F]), as for permutation
 * importance.  The K explained outputs of a window are at time step T-1 and column target_idx: pred_s of each stage
 * (K = S), tar_1, var_1, .., tar_S, var_S on a uq chain (K = 2S), pred[:, target_idx] on a dense handle (K = 1).
 * Sample m < samples belongs to pair p = m / 2: window i's donor is d_p(i) = lfmq_permutation_index(N, seed,
 * 0x40000000, p, i); an even sample orders the groups by o_m[q] = lfmq_permutation_index(G, seed, 0x40000001, p, q), an
 * odd one by the reverse of o_{m-1}.  Copy (m, k), k = 0..G, is x with the columns whose group ranks >= k in o_m taken
 * from window d_p(i) (k = 0: the donor, k = G: x itself).  Every launch of sample m keys window i as row m * N + i at
 * `step`: on a uq model all copies of a sample share window i's dropout masks, the ones lfmq_forward_uq_mc draws for
 * sample m at B = N; point and dense models predict with dropout off.  Outputs (device fp32):
 *   phi [N][K][G]: (1/M) sum_m f_m(copy (m, r + 1)) - f_m(copy (m, r)), r = the rank of g in o_m;
 *   f_x [N][K] = (1/M) sum_m f_m(copy (m, G)), f_bg [N][K] = (1/M) sum_m f_m(copy (m, 0)),
 * so sum_g phi = f_x - f_bg.  A window's terms are added in increasing (m, k) in fp64 without atomics and divided by M
 * at the end, so a point model's f_x is its forward bit for bit: the outputs do not depend on max_batch or on where
 * launches are cut.  Accepted: what
 * lfmq_chain_permutation_importance accepts.  The handles' parameters, gradient buffers (tail included) and optimizer
 * slots are left untouched.  N, G or samples < 1, a col_group value outside [0, G) or a null pointer: LFMQ_ERR_ARG.
 * `work`: caller-owned device scratch, 256-byte aligned, of the size the *_work_bytes query gives: one launch's rows
 * (per stage), the col_group copy, the orderings and ranks [samples][G], prev [N][K], the fp64 sums [N][K][G + 2] and
 * one launch's predictions (and variances). */
int32_t lfmq_chain_shapley_work_bytes(const lfmq_handle* stages, int32_t n_stages, int32_t N, int32_t G,
                                      int32_t samples, uint64_t* bytes);
int32_t lfmq_chain_shapley(const lfmq_handle* stages, int32_t n_stages, const float* x, int32_t N,
                           const int32_t* col_group, int32_t G, int32_t samples, uint64_t seed, int64_t step,
                           float* phi, float* f_x, float* f_bg, void* work, uint64_t work_bytes, void* stream);
/* ---- accumulated local effects -------------------------------------------------------------------------------------
 * In which direction and with what shape the forecast responds to single input columns (ALE, Apley & Zhu 2020).
 * x [N,T,F] (or [N,T*F] on a dense handle) are the model's inputs; feature g < G is column cols[g] in [0, T*F) (host
 * int32 [G]), c = t * F + f.  The J explained outputs are those of lfmq_chain_shapley (J = S, 2S on a uq chain, 1 on a
 * dense handle).  Per feature: v_i = x[i, cols[g]]; non-finite values are left out, N' counts the others.  With v_(1) <=
 * .. <= v_(N') sorted, the type-1 quantiles q_0 = v_(1), q_k = v_(ceil(k N' / K)) for k = 1..K with repeated values
 * dropped are the edges z_0 < .. < z_Kg, n_bins[g] = Kg <= K (0 with fewer than two distinct finite values).  Window i is
 * in bin k (1-based) when z_{k-1} < v_i <= z_k, or v_i = z_0 for k = 1; n_k windows are.  Its local effect d_i =
 * f(x_i with column cols[g] at z_k) - f(x_i with it at z_{k-1}), fp32, both copies keyed as row i at `step` (on a uq
 * model they share window i's dropout masks; point and dense models predict with dropout off).  Outputs (device):
 *   n_bins [G] int32; edges [G][K+1] fp32, z_k, NaN past Kg (and at 0 when N' = 0); counts [G][K] int32, n_k, 0 past Kg;
 *   local_mean [G][K][J] and local_sd [G][K][J]: the mean and population standard deviation of d over bin k;
 *   ale [G][K+1][J]: g(z_k) - (1/N') sum_k n_k (g(z_{k-1}) + g(z_k)) / 2 with g(z_0) = 0, g(z_k) = sum_{k'<=k}
 *   local_mean_k' (ALEPlot's centring: the count-weighted mean effect is 0).  Every float output is NaN past Kg, and
 *   ale, local_mean and local_sd are NaN throughout when Kg = 0.
 * The values are sorted per feature by a stable segmented radix sort (ties keep window order, -0 counts as +0); each
 * bin's sums run over its contiguous run of that order in fp64 in a fixed order, without atomics, so the outputs do not
 * depend on max_batch or on where launches are cut, and two calls give the same bits.  The call waits once for n_bins
 * on the host, to skip the copies of features without bins.  Accepted: what lfmq_chain_permutation_importance accepts.
 * The handles' parameters, gradient buffers (tail included) and optimizer slots are left untouched.  N, G or K < 1,
 * K > 1024, G * N >= 2^31, a column outside [0, T*F) or a null pointer: LFMQ_ERR_ARG.  `work`: caller-owned device
 * scratch, 256-byte aligned, of the size the *_work_bytes query gives: one launch's rows (per stage), the cols copy, the
 * sort's keys, windows and temp storage, the bin ends [G][K+1], every window's bin [G][N], d [N][J], the fp64 bin means
 * [K][J] and one launch's predictions (and variances). */
int32_t lfmq_chain_ale_work_bytes(const lfmq_handle* stages, int32_t n_stages, int32_t N, int32_t G, int32_t K,
                                  uint64_t* bytes);
int32_t lfmq_chain_ale(const lfmq_handle* stages, int32_t n_stages, const float* x, int32_t N, const int32_t* cols,
                       int32_t G, int32_t K, int64_t step, int32_t* n_bins, float* edges, int32_t* counts, float* ale,
                       float* local_mean, float* local_sd, void* work, uint64_t work_bytes, void* stream);
/* ---- training-window attributions -----------------------------------------------------------------------------------
 * Which training windows taught the model each forecast: TracIn (Pruthi et al. 2020) at the trained checkpoint,
 * restricted to the output head theta (OUTPUT_1, or OUTPUT_TARGET_1 and OUTPUT_VARIANCE_1), with every dropout off.
 * The influence of training window t on output j of query window q is I_j(t, q) = -grad_theta l_t . grad_theta f^j_q,
 * the first-order change of the forecast from one unit-rate gradient step on t alone: positive pushes it up.  l_t is
 * the training loss of a batch holding t alone (B = 1, the window's own mask counts as denominators, no row weights;
 * masked all-zero-target elements contribute exactly 0).  The J outputs are pred[T-1, target_idx] (J = 1) and on a uq
 * handle also the variance (J = 2).  With a_tau the head input at step tau (the last layer's output after
 * BatchNormalization, D = num_hidden; on a dense handle the flattened window, D = T * F, one step) and ~a = (a; 1):
 *   I_j(t, q) = -s_jq (~a_{q,T-1} . u_jt),  u_jt = sum_tau G_j[t, tau] ~a_{t,tau}  (length D1 = D + 1)
 * where G_j = dl_t / d(head output j at [tau, target_idx]) (the variance head's pre-softplus activation), s_0q = 1 and
 * s_1q = sigmoid(pre_q), 0 where the 1e-6 variance floor binds.
 * lfmq_influence_train_features: u [J][B][D1] of B training windows x, y.
 * lfmq_influence_query_features: ~a [B][D1] and s [J][B] of B query windows.
 * Both run a forward with every dropout off (also on a uq handle) in launches of at most max_batch rows (B is not
 * bounded by it), with the training loss's device expressions.  Accepted: recurrent handles of precision LFMQ_PREC_FP32
 * or LFMQ_PREC_TF32 (either cell, point or uq, forward_only or not) and dense handles; one handle, so a forecast chain
 * is not accepted.  LFMQ_PREC_BF16 / LFMQ_PREC_BF16X3 handles, B < 1 and null pointers: LFMQ_ERR_ARG (explain a
 * LFMQ_PREC_FP32 handle with the same parameters).  Parameters, gradients and optimizer slots are left untouched.
 * `work`: caller-owned device scratch, 256-byte aligned, of the size lfmq_influence_features_work_bytes gives. */
int32_t lfmq_influence_features_work_bytes(lfmq_handle h, uint64_t* bytes);
int32_t lfmq_influence_train_features(lfmq_handle h, const float* x, const float* y, int32_t B, float* u, void* work,
                                      uint64_t work_bytes, void* stream);
int32_t lfmq_influence_query_features(lfmq_handle h, const float* x, int32_t B, float* a, float* s, void* work,
                                      uint64_t work_bytes, void* stream);
/* Per query q and output j, from a [Nq][D1], u [J][Nt][D1] and s [J][Nq] (device fp32; no handle):
 *   pos_idx / pos_score [Nq][J][K]  the K largest positive influences, largest first
 *   neg_idx / neg_score [Nq][J][K]  the K most negative, most negative first
 *   total [Nq][J]                   sum_t I_j(t, q) over the whole pool
 * Ties go to the lower training index; fewer than K influences of a sign pad the list with index -1 and score 0 (a zero
 * influence has no sign).  The scores a . u run on sm_90a wgmma with every operand split into tf32 high and low parts
 * (hi*hi + hi*lo + lo*hi, fp32 accumulation: about 1e-6 |a| |u| of fp64), each over its k range in a fixed order, and
 * the top K is kept exactly inside the GEMM's epilogue, per pool slice, then merged.  total is -s (a . sum_t u_t) with
 * the sum and the product in fp64 in a fixed order.  Two calls give the same bits, and a query's results do not depend
 * on Nq, on the other queries or on the pool split.  1 <= K <= 64, J in {1, 2}, Nq, Nt, D1 >= 1, else LFMQ_ERR_ARG, as
 * for null pointers.  `work`: device scratch, 256-byte aligned, of the size lfmq_influence_topk_work_bytes gives. */
int32_t lfmq_influence_topk_work_bytes(int32_t Nq, int32_t Nt, int32_t D1, int32_t J, int32_t K, uint64_t* bytes);
int32_t lfmq_influence_topk(const float* a, const float* u, const float* s, int32_t Nq, int32_t Nt, int32_t D1,
                            int32_t J, int32_t K, int32_t* pos_idx, float* pos_score, int32_t* neg_idx,
                            float* neg_score, float* total, void* work, uint64_t work_bytes, void* stream);
/* ---- nearest pool rows ----------------------------------------------------------------------------------------------
 * The K rows of the pool b [Nt][D1] nearest to each query a [Nq][D1] in Euclidean distance (device fp32; no handle):
 *   idx [Nq][K]  pool rows, nearest first, ties to the lower index; -1 past Nt
 *   d2 [Nq][K]   |a - b|^2, summed from the difference in fp64 and rounded to fp32; +inf past Nt
 *   mean [Nq]    with value [Nt]: the mean of value over the listed rows, summed in rank order in fp64
 * It is lfmq_influence_topk's kernel in a second mode: the same 3xTF32 wgmma product a.b, scored 2 a.b - |b|^2 (|b|^2
 * summed in fp64 in a fixed order and rounded to fp32), with one list of the largest scores kept in the epilogue.  That
 * score shortlists K + 16 rows per query; their exact fp64 distances then pick and order the K (the score alone
 * cannot resolve a small distance next to large norms: its fp32 accumulation errs by about 1e-5 (|a|^2 + |b|^2) at
 * D1 ~ 1500).  A row missing from the result is at most the score's error nearer than the K-th listed one; two calls
 * give the same bits, and a query's results do not depend on Nq, on the other queries or on the pool split.
 * 1 <= K <= 64, Nq, Nt, D1 >= 1, else LFMQ_ERR_ARG, as for null pointers (value and mean are both given or both null).
 * `work`: device scratch, 256-byte aligned, of the size lfmq_nearest_topk_work_bytes gives. */
int32_t lfmq_nearest_topk_work_bytes(int32_t Nq, int32_t Nt, int32_t D1, int32_t K, uint64_t* bytes);
int32_t lfmq_nearest_topk(const float* a, const float* b, const float* value, int32_t Nq, int32_t Nt, int32_t D1,
                          int32_t K, int32_t* idx, float* d2, float* mean, void* work, uint64_t work_bytes,
                          void* stream);
/* ---- split-conformal prediction intervals ---------------------------------------------------------------------------
 * DESIGN.md section 5j.  Arrays are device fp32 [S][N] (S forecast steps, N windows; no handle), so any model, the
 * naive forecast included, uses the same calls.  The nonconformity score of a window with a finite target y is
 *   r = |y - pred| / scale        (scale optional: 1 when null; it must be > 0)
 * in IEEE single precision, subtraction and division each rounded once: the bits NumPy's float32 arithmetic gives.
 * r is NaN where y is not finite.  scale is sigma for a UQ forecast, d(x) + beta for the normalised kNN score, or null.
 * lfmq_conformal_scores: r [S][N].
 * lfmq_conformal_calibrate: of the calibration windows [S][Nc] and the host fp64 levels l_1 < .. < l_Q in (0, 1),
 * Q <= 32:
 *   n_valid [S]       the windows of step s with a score (finite target)
 *   sorted [S][Nc]    step s's scores ascending, NaN after the n_valid[s] scores (one radix sort of every step)
 *   qhat [S][Q]       the ceil((n + 1) l)-th smallest score (rank in fp64), +inf when that rank exceeds n = n_valid[s]
 * lfmq_conformal_apply: of the query windows [S][N] (y optional), with calibrate's outputs:
 *   lower / upper [S][N][Q]  pred -/+ qhat * scale (product and sum each rounded once; +-inf where qhat is +inf)
 *   pvalue [S][N]            (1 + #{i : r_i >= r}) / (n + 1) by binary search in sorted; NaN where y is null or not
 *                            finite
 * S, N, Nc >= 1 with S * N and S * Nc below 2^31, levels as above, and null pointers (other than y and scale):
 * LFMQ_ERR_ARG.  The results do not depend on the order of the windows.  `work`: device scratch, 256-byte aligned, of
 * the size the call's *_work_bytes gives (0 bytes for scores and apply). */
int32_t lfmq_conformal_scores_work_bytes(int32_t S, int32_t N, uint64_t* bytes);
int32_t lfmq_conformal_scores(const float* pred, const float* y, const float* scale, int32_t S, int32_t N, float* r,
                              void* work, uint64_t work_bytes, void* stream);
int32_t lfmq_conformal_calibrate_work_bytes(int32_t S, int32_t Nc, uint64_t* bytes);
int32_t lfmq_conformal_calibrate(const float* pred, const float* y, const float* scale, int32_t S, int32_t Nc,
                                 const double* levels, int32_t Q, int32_t* n_valid, float* sorted, float* qhat,
                                 void* work, uint64_t work_bytes, void* stream);
int32_t lfmq_conformal_apply_work_bytes(int32_t S, int32_t N, int32_t Nc, int32_t Q, uint64_t* bytes);
int32_t lfmq_conformal_apply(const float* pred, const float* y, const float* scale, int32_t S, int32_t N,
                             const float* sorted, const int32_t* n_valid, const float* qhat, int32_t Nc, int32_t Q,
                             float* lower, float* upper, float* pvalue, void* work, uint64_t work_bytes,
                             void* stream);
/* ---- lookahead factor backtests -------------------------------------------------------------------------------------
 * DESIGN.md section 5k.  N rows, each with a date index date_idx [N] in [0, D) and a company code company [N] (device
 * int32; no two rows share a (date, company) pair), G factor scores score [G][N] and M outcome measures measure [M][N]
 * (device fp64; no handle, so every model, the naive forecast included, uses the one call).  For factor g and date d
 * the universe is the rows of d with a finite score; each gets its average rank r among them (ties share the mean
 * rank; -0 ties +0) and the bucket floor((r - 1/2) Q / n) + 1 in [1, Q], bucket Q the highest scores.  Outputs:
 *   n [G][D]                the universe's size
 *   bucket_n [G][D][Q]      the rows of each bucket
 *   n_pair [G][M][D]        the rows of d where score and measure are both finite
 *   ic [G][M][D]            Spearman's rank correlation over those rows (both re-ranked over them; NaN when
 *                           n_pair < 3 or either rank variance is 0), from exact integer rank moments
 *   bucket_mean [G][M][D][Q] the mean measure of each bucket's rows with a finite measure (NaN when none)
 *   spread [G][M][D]        bucket_mean of bucket Q - bucket_mean of bucket 1
 *   turnover [G][D]         the share of bucket Q's companies at d that were not in bucket Q at date index d - 1;
 *                           NaN at d = 0 or when bucket Q is empty
 * Every fp64 sum runs over a date in (score, company) order, with no atomics: permuting the rows, or calling twice,
 * gives the same bits.  N, D >= 1, 1 <= G <= 8, 1 <= M <= 4, 2 <= Q <= 100 and null pointers: LFMQ_ERR_ARG.  The call
 * does not synchronise with the host.  `work`: device scratch, 256-byte aligned, of the size
 * lfmq_factor_eval_work_bytes gives. */
int32_t lfmq_factor_eval_work_bytes(int32_t N, int32_t D, int32_t G, int32_t M, int32_t Q, uint64_t* bytes);
int32_t lfmq_factor_eval(const int32_t* date_idx, const int32_t* company, int32_t N, int32_t D, const double* score,
                         int32_t G, const double* measure, int32_t M, int32_t Q, int32_t* n, int32_t* bucket_n,
                         int32_t* n_pair, double* ic, double* bucket_mean, double* spread, double* turnover, void* work,
                         uint64_t work_bytes, void* stream);
/* uq chain: Losses.weight_adjusted_uq_loss(y_true list, y_pred list, y_var list) (losses.py:137-178): out_dev =
 * {sum_s w_s uq_loss_s, sum_s w_s uq_loss_last_tar_s, sum_s w_s mse_s}, each stage with its own mask counts.  A
 * zero-padded step makes the uq loss NaN, as for lfmq_loss_uq.  B may exceed max_batch (validation). */
int32_t lfmq_chain_loss_uq(const lfmq_handle* stages, int32_t n_stages, const float* const* preds,
                           const float* const* vars, const float* const* y, const float* weights, int32_t B,
                           float* out_dev, void* stream);
/* forward of all stages, the weighted loss, and BPTT through the whole graph: the input gradient of stage s flows into
 * the last time step of the earlier predictions it was built from.  Fills every stage's gradient buffer;
 * loss_out_dev (nullable) = {loss, mse} as lfmq_chain_loss; on a uq chain (3 floats) {uq_loss, uq_loss_last_tar, mse}
 * as lfmq_chain_loss_uq, the gradient of sum_s w_s uq_loss_s (train.py:201-218). */
int32_t lfmq_chain_backward(const lfmq_handle* stages, int32_t n_stages, const float* x, const float* const* y,
                            const float* weights, int32_t B, int64_t row0, int64_t step, float* work,
                            float* loss_out_dev, void* stream);
/* tf.clip_by_global_norm over the variables of ALL stages (train.py:195-196, stage 0's max_grad_norm), then each
 * stage's optimizer update and MaxNorm constraint. */
int32_t lfmq_chain_apply(const lfmq_handle* stages, int32_t n_stages, float lr, int64_t iteration, void* stream);

/* ---- data parallelism over the company-batch axis for chains and uq handles ----
 * Each rank runs the chain's backward on its rows with the loss denominators of the whole global batch, packs every
 * stage's gradients and loss tail into one contiguous vector, all-reduces it (SUM, the only collective of the step),
 * unpacks it and runs lfmq_chain_apply (or lfmq_apply on a single handle), which clips, updates and constrains the
 * same reduced gradients on every rank.  A rank without rows packs nothing: it zeroes the vector and joins the
 * all-reduce, the unpack and the apply. */
/* Every stage's counts for one batch: out_dev[3 s .. 3 s + 2] = {B, sum(mask), sum(mask[:, T-1])} of y[s], as
 * lfmq_mask_count_uq.  The host all-reduces the 3 * n_stages floats once per batch.  Point and uq chains alike. */
int32_t lfmq_chain_mask_count(const lfmq_handle* stages, int32_t n_stages, const float* const* y, int32_t B,
                              float* out_dev, void* stream);
/* lfmq_chain_backward with the stages' counts of the global batch (lfmq_chain_mask_count summed over the ranks,
 * device, 3 floats per stage) as every loss denominator.  row0 = global index of this shard's first row (keys the
 * dropout masks).  Each stage's tail and loss_out_dev then hold this shard's contributions to the global values. */
int32_t lfmq_chain_backward_dp(const lfmq_handle* stages, int32_t n_stages, const float* x, const float* const* y,
                               const float* weights, int32_t B, int64_t row0, int64_t step, const float* denom_dev,
                               float* work, float* loss_out_dev, void* stream);
/* Length of the packed vector: sum_s (n_trainable_s + k), k = 2 tail entries {loss, mse_0} on a point-estimate chain,
 * k = 3 {uq_loss, mse_0, uq_loss_last_tar} on a uq chain.  grad_norm and clip_scale are not carried: the apply computes
 * them from the reduced gradients. */
int32_t lfmq_chain_grad_pack_size(const lfmq_handle* stages, int32_t n_stages, int64_t* n_elems);
/* flat (device, 16-byte aligned) = [grads_0[0:n_0], tail_0, grads_1[0:n_1], tail_1, ...]: one launch for all stages */
int32_t lfmq_chain_grad_pack(const lfmq_handle* stages, int32_t n_stages, float* flat, void* stream);
/* The inverse scatter into the stages' gradient buffers.  loss_out_dev (nullable; needs the host `weights`) = the
 * weighted sums over the stages of the unpacked tails, as lfmq_chain_backward's loss_out_dev. */
int32_t lfmq_chain_grad_unpack(const lfmq_handle* stages, int32_t n_stages, const float* flat, const float* weights,
                               float* loss_out_dev, void* stream);

/* Dataset.get_batch (data_processing.py:307-368) with _get_train_seq/_get_pred_seq (:370-449) and
 * log_squasher (:600-609) over a device-resident float64 copy of Dataset.data_values' numeric columns.
 *   table [n_rows, n_cols] f64; inp_idx/tar_idx [B,3] int32 (start, end, pad) (data_processing.py:267-279)
 *   inp_cols [F], fin_cols [O] int32 column ids; seq_norm_col < 0 when there is no scale field
 *   center/scale [>=F] f64 (scaling_params, :352-357); scale_flag [F] u8 = column in scale_inp_col_ids;
 *   aux_flag [F] u8 = aux column zeroed for t < T-1 when aux_masking (:359-361)
 * Outputs x [B,T,F] f32, y [B,T,O] f32 (NaN where the target row does not exist, :427-435),
 * seq_norm [B] f64 (:393-396).  Arithmetic is fp64 then cast, as the reference. */
typedef struct lfmq_gather_args {
  int32_t struct_size;
  int32_t n_rows, n_cols, B, T, F, O, stride, seq_norm_col, log_squasher, aux_masking;
  const double* table;
  const int32_t* inp_idx;
  const int32_t* tar_idx;
  const int32_t* inp_cols;
  const int32_t* fin_cols;
  const double* center;
  const double* scale;
  const uint8_t* scale_flag;
  const uint8_t* aux_flag;
  float* x;
  float* y;
  double* seq_norm;
} lfmq_gather_args;
int32_t lfmq_gather_batch(const lfmq_gather_args* args, void* stream);
/* The row weights of one training batch for lfmq_set_row_weights (DESIGN.md section 6d), from the same fp64 table
 * [n_rows, n_cols] and the batch's input triples inp_idx [B][3] (row 1 of a triple is the window's last input row, its
 * forecast origin).  w_out[b] = fp32 of the fp64 product of the enabled sources: table[row][weight_col] with NaN as 0
 * (weight_col >= 0), and 2^(-months / (12 halflife_years)) (halflife_years > 0), where months = ref_month - (12 year +
 * month) of the yyyymmdd date in table[row][date_col].  At least one source must be enabled. */
int32_t lfmq_row_weights(const double* table, int64_t n_rows, int32_t n_cols, const int32_t* inp_idx, int32_t B,
                         int32_t weight_col, int32_t date_col, double halflife_years, int32_t ref_month, float* w_out,
                         void* stream);

/* Dataset._create_tf_dataset + _append_sequence_data (data_processing.py:170-305) on the device: the window index
 * triples (start, end, pad) of every table row that yields a window, in row order.
 *   key [n] int32: any code with key[i] == key[j] <=> same gvkey (rows of one company are consecutive, :203-219)
 *   active [n] u8 (:211); date [n] int32 in any order-preserving encoding (yyyymmdd), compared with start_date,
 *   end_date and last_train_date = end_date - stride months (:221-234); train selects the training rule (:221-225:
 *   the target row forecast_n rows ahead must belong to the same key) or the prediction rule (:231-234)
 *   min_unrollings / max_unrollings / stride / forecast_n as the flags of that name (:263-279)
 * Outputs (device): inp_idx, tar_idx int32 [cap][3], rows int32 [cap] (table row of each window), count int32 [1]
 * (the number of windows; entries beyond cap are dropped -- size cap = n to be safe).
 * work: device ints, 4 * ceil(n / 1024) + n. */
typedef struct lfmq_window_index_args {
  int32_t struct_size;
  int32_t n, train, stride, forecast_n, min_unrollings, max_unrollings;
  int32_t start_date, end_date, last_train_date;
  int32_t cap;
  const int32_t* key;
  const uint8_t* active;
  const int32_t* date;
  int32_t* inp_idx;
  int32_t* tar_idx;
  int32_t* rows;
  int32_t* count;
  int32_t* work;
} lfmq_window_index_args;
int32_t lfmq_window_index(const lfmq_window_index_args* args, void* stream);

/* Train._unscale_preds (train.py:420-432) on the device, for the validation pass (train.py:268-336) without a host
 * round trip: out[r][k] = reverse_log_squasher(in[r][k] * scale[k] + center[k]) (data_processing.py:611-619), fp64
 * arithmetic then cast to fp32 as the reference's NumPy expression does.  in/out [n_rows][O] fp32 (may alias),
 * scale/center [>= O] fp64 device arrays (Dataset.scaling_params). */
int32_t lfmq_unscale(const float* in, float* out, int64_t n_rows, int32_t O, const double* scale, const double* center,
                     int32_t log_squasher, void* stream);

/* Instrumentation: number of kernels this library has launched since load (bench.py "gpu_launches"). */
int64_t lfmq_launch_count(void);

/* Instrumentation for bench.py's roofline: while enabled, each region of a step is bracketed by CUDA events
 * recorded on the caller's stream (at most 256 occurrences per region are kept between reads).
 * lfmq_profile_enable(h, 1) also resets the counters; lfmq_profile_read synchronises the recorded events and
 * returns the summed device time and the number of occurrences of `region`. */
enum { LFMQ_REGION_FWD = 0,   /* LSTM recurrence (+BN/dropout) forward, all layers */
       LFMQ_REGION_HEAD = 1,  /* Dense head + loss (+ their gradients) */
       LFMQ_REGION_BWD = 2,   /* LSTM recurrence backward (dz, dh chain) */
       LFMQ_REGION_WGRAD = 3, /* batched weight-gradient GEMMs (dW, dU, db, dx) */
       LFMQ_REGION_OPT = 4,   /* clip + optimizer + MaxNorm */
       LFMQ_N_REGIONS = 5 };
int32_t lfmq_profile_enable(lfmq_handle h, int32_t enable);
int32_t lfmq_profile_read(lfmq_handle h, int32_t region, float* total_ms, int32_t* count);

#ifdef __cplusplus
}
#endif
#endif /* LFMQ_H_ */
