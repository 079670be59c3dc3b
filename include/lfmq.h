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
 *     (thread-local).  One handle per process/GPU; a handle is not thread-safe.
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
 * LFMQ_PREC_BF16:   gate GEMMs on wgmma tensor cores with bf16 operands, fp32 accumulate, fp32 cell state.  LSTM cell,
 *                   point-estimate head, num_hidden a multiple of 64 (<= 1024), any num_layers, dropout and recurrent
 *                   dropout; H = 256 / L = 1 without recurrent dropout runs the persistent cluster kernels.
 * LFMQ_PREC_BF16X3: fp32-tolerance forward on tensor cores (forward_only handles: predict.py:129): every operand split
 *                   into bf16 high + low halves, three wgmma products per GEMM (hi*hi + lo*hi + hi*lo), accurate
 *                   expf / tanhf gate nonlinearities, fp32 head -- <=1e-4 rel vs the oracle. */
enum { LFMQ_PREC_FP32 = 0, LFMQ_PREC_BF16 = 1, LFMQ_PREC_BF16X3 = 2 };

/* config.rnn_cell (lfm_quant.py:39; rnn_point_estimate.py:80-102).  GRU is Keras' default reset_after=True cell:
 * 3 gate blocks z|r|h, bias [2][3H] (input row, recurrent row).  LFMQ_PREC_BF16 supports the LSTM cell only. */
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

/* model.trainable_variables / model.weights (train.py:192,198): tensors are listed in Keras order,
 * trainable ones first: per layer lstm_l/{kernel,recurrent_kernel,bias} (gru_l/... with bias [2][3H] for LFMQ_CELL_GRU), batch_normalization[_k]/{gamma,beta};
 * OUTPUT_1/{kernel,bias} (uq: OUTPUT_TARGET_1/{kernel,bias}, OUTPUT_VARIANCE_1/{kernel,bias}); then per layer batch_normalization[_k]/{moving_mean,moving_variance}. */
int32_t lfmq_param_count(lfmq_handle h, int32_t* n_tensors, int64_t* n_trainable_elems, int64_t* n_total_elems);
int32_t lfmq_param_spec(lfmq_handle h, int32_t index, char* name, int32_t name_cap, int32_t* ndim,
                        int64_t shape[2], int64_t* offset_elems, int32_t* trainable);
/* Device pointers into the workspace: flat fp32 parameters [n_total]; flat gradients
 * [n_trainable + 8] whose tail holds {loss, mse_0} contributions of the last lfmq_backward,
 * {grad_norm, clip_scale} of the last lfmq_apply and, on a uq handle, [4] = uq_loss_last_tar (tail[0] is then the
 * weighted uq loss); optimizer slots [n_slots * n_trainable]. */
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

/* First half of Train._train_step_point (train.py:181-192): forward, loss, BPTT.  Fills the flat
 * gradient buffer (+ its 4-float tail).  denom_dev = device {B_global, mask_count_global} or NULL to use
 * this call's own batch.  With N ranks the host all-reduces grads[0 : n_trainable+2] (SUM) next.
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
 * Training-mode stages (cfg.train) run on the LFMQ_PREC_FP32 kernels; forward_only stages may use any precision. */
/* model(inp) -> [pred_1 .. pred_S], each [B,T,O] (train.py:182, predict.py:129) */
int32_t lfmq_chain_forward(const lfmq_handle* stages, int32_t n_stages, const float* x, int32_t B, int64_t row0,
                           int64_t step, float* const* preds, float* work, void* stream);
/* Losses.weight_adjusted_mse(y_true list, y_pred list) (losses.py:19-53): out_dev = {sum_s w_s loss_s, sum_s w_s mse_s} */
int32_t lfmq_chain_loss(const lfmq_handle* stages, int32_t n_stages, const float* const* preds, const float* const* y,
                        const float* weights, int32_t B, float* out_dev, void* stream);
/* forward of all stages, the weighted loss, and BPTT through the whole graph: the input gradient of stage s flows into
 * the last time step of the earlier predictions it was built from.  Fills every stage's gradient buffer;
 * loss_out_dev (nullable) = {loss, mse} as lfmq_chain_loss. */
int32_t lfmq_chain_backward(const lfmq_handle* stages, int32_t n_stages, const float* x, const float* const* y,
                            const float* weights, int32_t B, int64_t row0, int64_t step, float* work,
                            float* loss_out_dev, void* stream);
/* tf.clip_by_global_norm over the variables of ALL stages (train.py:195-196, stage 0's max_grad_norm), then each
 * stage's optimizer update and MaxNorm constraint. */
int32_t lfmq_chain_apply(const lfmq_handle* stages, int32_t n_stages, float lr, int64_t iteration, void* stream);

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
