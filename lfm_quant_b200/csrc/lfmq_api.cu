// C-ABI entry points (include/lfmq.h) and step orchestration.
#include "../../include/lfmq.h"

#include <math.h>
#include <stdlib.h>
#include <string.h>

#include <algorithm>
#include <memory>
#include <string>
#include <vector>

#include "dense.h"
#include "kernels.h"
#include "lstm_tc.h"
#include "rnn_tc.h"

using namespace lfmq;

namespace {

struct ParamSpec {
  std::string name;
  int ndim;
  int64_t shape[2];
  int64_t offset;
  int trainable;
};

// The fp32 path's activations of one layer
struct LayerBuf {
  float *h, *c, *y, *gates, *rmask;
};

// The code that runs a handle, chosen once at create (choose_path).  Fp32 is the fp32 step (forward_fp32 /
// backward_fp32) of LFMQ_PREC_FP32 and LFMQ_PREC_TF32 handles (gemm() picks the GEMM); Cluster the persistent cluster
// kernels (lstm_tc.cu); General the general stepped tensor-core path (rnn_tc.cu); Dense the linear model (dense.cu).
enum class Path { Fp32, Cluster, General, Dense };

// The handle's block of device scalars (zeroed at create).  Each user resets the tickets it used.
struct Scalars {
  unsigned int mask_tickets[2];   // mask_count: the count and the last-block ticket
  unsigned int norm_ticket;       // grad_norm_scale
  unsigned int unused0[5];
  float denom[3];                 // the loss counts of the handle's own batch (mask_count, stages_loss_uq)
  float unused1;
  float chain_loss[2];            // lfmq_chain_loss: this stage's {loss, mse}
  float unused2[2];
};
static_assert(sizeof(Scalars) == 16 * sizeof(float), "one 64-byte block");

}  // namespace

struct lfmq_handle_s {
  lfmq_config cfg;
  Path path = Path::Fp32;
  std::vector<ParamSpec> specs;
  lfmq::ParamLayout pl;      // offsets of the specs' tensors
  int64_t n_train = 0, n_total = 0, n_grad_buf = 0;
  int n_slots = 0;
  // workspace carve
  float *params = nullptr, *grads = nullptr, *slots = nullptr, *scratch = nullptr;
  Scalars* sc = nullptr;
  size_t scratch_elems = 0;
  // the fp32 path's activations
  std::vector<LayerBuf> layers;
  float *z = nullptr, *hm = nullptr, *dz = nullptr, *dy = nullptr, *dh_out = nullptr, *hp = nullptr;
  float *dh_rec = nullptr, *dc = nullptr, *dpred = nullptr, *preds = nullptr;
  // uq only: variance output, its pre-activation, gradient w.r.t. the pre-activation
  float *var = nullptr, *apre = nullptr, *da = nullptr;
  // GRU only: recurrent projection of one step, gradient w.r.t. the recurrent projection
  float *zh = nullptr, *dz2 = nullptr;
  lfmq::TcState tc;
  int64_t last_step = 0;     // step and row0 of the last forward: the fp32 backward regenerates that call's dropout masks
  int64_t last_row0 = 0;
  lfmq::Profiler prof;
  // the linear baseline (lfmq_dense_create): cfg carries its shapes, target, loss weight, optimizer and clip, with
  // num_layers = 0; preds / dpred are its [B, O] outputs and their gradient
  int huber = 0;
  float huber_delta = 1.f;
  float* wpart = nullptr;    // row-block partials of the weight gradient (dense_wgrad)

  ~lfmq_handle_s() {
    lfmq::tc_destroy(tc);
    lfmq::gen_destroy(tc);
    if (prof.created)
      for (int r = 0; r < lfmq::Profiler::kRegions; ++r)
        for (int i = 0; i < lfmq::Profiler::kCap; ++i) {
          cudaEventDestroy(prof.a[r][i]);
          cudaEventDestroy(prof.b[r][i]);
        }
  }
};

namespace {

int validate(const lfmq_config* c) {
  if (!c || c->struct_size != (int32_t)sizeof(lfmq_config)) {
    LFMQ_SET_ERR("lfmq_config: struct_size mismatch (got %d, want %zu)", c ? c->struct_size : -1, sizeof(lfmq_config));
    return LFMQ_ERR_ARG;
  }
  if (c->max_batch <= 0 || c->seq_len <= 0 || c->n_inputs <= 0 || c->n_outputs <= 0 || c->num_hidden <= 0 ||
      c->num_layers <= 0) {
    LFMQ_SET_ERR("lfmq_config: non-positive dimension");
    return LFMQ_ERR_ARG;
  }
  if (c->num_hidden % 4 != 0 || c->num_hidden > 1024) {
    LFMQ_SET_ERR("lfmq_config: num_hidden must be a multiple of 4 and <= 1024 (got %d)", c->num_hidden);
    return LFMQ_ERR_UNSUPPORTED;
  }
  if (c->target_idx < 0 || c->target_idx >= c->n_outputs) {
    LFMQ_SET_ERR("lfmq_config: target_idx %d outside [0,%d)", c->target_idx, c->n_outputs);
    return LFMQ_ERR_ARG;
  }
  if (c->optimizer < 0 || c->optimizer > 3) {
    LFMQ_SET_ERR("lfmq_config: unknown optimizer %d", c->optimizer);
    return LFMQ_ERR_ARG;
  }
  if (c->dropout < 0.f || c->dropout >= 1.f || c->recurrent_dropout < 0.f || c->recurrent_dropout >= 1.f) {
    LFMQ_SET_ERR("lfmq_config: dropout rates must be in [0,1)");
    return LFMQ_ERR_ARG;
  }
  if ((c->rnn_cell != LFMQ_CELL_LSTM && c->rnn_cell != LFMQ_CELL_GRU) || (c->uq != 0 && c->uq != 1)) {
    LFMQ_SET_ERR("lfmq_config: rnn_cell must be LFMQ_CELL_LSTM or LFMQ_CELL_GRU and uq 0 or 1 (got %d, %d)", c->rnn_cell,
                 c->uq);
    return LFMQ_ERR_ARG;
  }
  if (c->precision != LFMQ_PREC_FP32 && c->precision != LFMQ_PREC_BF16 && c->precision != LFMQ_PREC_BF16X3 &&
      c->precision != LFMQ_PREC_TF32) {
    LFMQ_SET_ERR("lfmq_config: unknown precision %d", c->precision);
    return LFMQ_ERR_ARG;
  }
  return LFMQ_OK;
}

// The one place that decides which code runs a recurrent handle: the fp32 step for LFMQ_PREC_FP32 and LFMQ_PREC_TF32;
// for LFMQ_PREC_BF16 the persistent cluster kernels on the shape family they are built for (LFMQ_FORCE_GENERIC=1 sends
// that family to the general path as well); the general path for every other tensor-core configuration it supports.
// Anything else is LFMQ_ERR_UNSUPPORTED, with *path = General.
int choose_path(const lfmq_config& c, Path* path) {
  char why[160];
  const char* fg = getenv("LFMQ_FORCE_GENERIC");
  const bool force_gen = fg != nullptr && atoi(fg) != 0;
  if (c.precision == LFMQ_PREC_FP32 || c.precision == LFMQ_PREC_TF32) {
    *path = Path::Fp32;
  } else if (c.precision == LFMQ_PREC_BF16 && !force_gen && lfmq::tc_supported(c, why, sizeof(why))) {
    *path = Path::Cluster;
  } else {
    *path = Path::General;
    if (!lfmq::gen_supported(c, why, sizeof(why))) {
      LFMQ_SET_ERR("tensor-core precision unsupported for this configuration: %s; use LFMQ_PREC_FP32", why);
      return LFMQ_ERR_UNSUPPORTED;
    }
  }
  return 0;
}

// The parameter specs in Keras order, with their offsets in h->pl, and the workspace carve: parameters, gradients,
// optimizer slots, scalars and scratch, then the buffers of h->path (with_path = false leaves those out: the size of a
// configuration no path supports, which lfmq_create refuses).  With base == nullptr only sizes are computed.
size_t layout(lfmq_handle_s* h, char* base, bool with_path) {
  const lfmq_config& c = h->cfg;
  const int H = c.num_hidden, L = c.num_layers, T = c.seq_len, O = c.n_outputs;
  const size_t B = (size_t)c.max_batch, BT = B * T;
  const bool gru = c.rnn_cell == LFMQ_CELL_GRU;
  lfmq::ParamLayout& pl = h->pl;
  pl = lfmq::ParamLayout{};
  h->specs.clear();
  int64_t off = 0;
  auto add = [&](const std::string& name, int ndim, int64_t s0, int64_t s1, int trainable) {
    h->specs.push_back(ParamSpec{name, ndim, {s0, s1}, off, trainable});
    off += s0 * (ndim == 2 ? s1 : 1);
    return h->specs.back().offset;
  };
  auto bn = [](int l) {
    return l == 0 ? std::string("batch_normalization") : "batch_normalization_" + std::to_string(l);
  };
  pl.layers.resize(L);       // none on a dense handle
  for (int l = 0; l < L; ++l) {
    lfmq::ParamLayout::Layer& o = pl.layers[l];
    o.I = (l == 0) ? c.n_inputs : H;
    const int NG = gru ? 3 : 4;
    const std::string ls = std::string(gru ? "gru_" : "lstm_") + std::to_string(l + 1);
    o.oW = add(ls + "/kernel", 2, o.I, NG * H, 1);
    o.oU = add(ls + "/recurrent_kernel", 2, H, NG * H, 1);
    o.ob = gru ? add(ls + "/bias", 2, 2, 3 * H, 1) : add(ls + "/bias", 1, 4 * H, 1, 1);
    o.ogamma = add(bn(l) + "/gamma", 1, H, 1, 1);
    o.obeta = add(bn(l) + "/beta", 1, H, 1, 1);
  }
  if (c.uq) {
    pl.oWo = add("OUTPUT_TARGET_1/kernel", 2, H, O, 1);
    pl.obo = add("OUTPUT_TARGET_1/bias", 1, O, 1, 1);
    pl.oWv = add("OUTPUT_VARIANCE_1/kernel", 2, H, O, 1);
    pl.obv = add("OUTPUT_VARIANCE_1/bias", 1, O, 1, 1);
  } else {       // the dense model's OUTPUT_1 reads the flattened input window
    pl.oWo = add("OUTPUT_1/kernel", 2, h->path == Path::Dense ? (int64_t)T * c.n_inputs : H, O, 1);
    pl.obo = add("OUTPUT_1/bias", 1, O, 1, 1);
  }
  h->n_train = off;
  for (int l = 0; l < L; ++l) {
    pl.layers[l].omean = add(bn(l) + "/moving_mean", 1, H, 1, 0);
    pl.layers[l].ovar = add(bn(l) + "/moving_variance", 1, H, 1, 0);
  }
  h->n_total = off;
  h->n_grad_buf = (h->n_train + LFMQ_TAIL_LEN + 3) / 4 * 4;
  h->n_slots = (c.optimizer == LFMQ_OPT_ADADELTA || c.optimizer == LFMQ_OPT_ADAM) ? 2 : 1;

  Carver cv{base, 0};
  h->params = cv.take<float>(h->n_total);
  h->grads = cv.take<float>(h->n_grad_buf);
  h->slots = c.forward_only ? nullptr : cv.take<float>((size_t)h->n_slots * h->n_train);
  h->sc = cv.take<Scalars>(1);
  // scratch serves every path (lfmq_loss, grad_norm_scale; the fp32 BN backward)
  h->scratch_elems = (size_t)4 << 20;
  if (!c.forward_only && h->path != Path::Dense)
    h->scratch_elems = std::max(h->scratch_elems, ((BT + 127) / 128) * 2 * H + (size_t)1024 * 2 * H);
  h->scratch = cv.take<float>(h->scratch_elems);
  if (!with_path) return cv.off;
  switch (h->path) {
    case Path::Fp32:
      h->layers.assign(L, LayerBuf{});
      for (LayerBuf& lb : h->layers) {
        lb.h = cv.take<float>(BT * H);
        lb.c = cv.take<float>(BT * H);
        lb.y = cv.take<float>(BT * H);
        lb.gates = c.forward_only ? nullptr : cv.take<float>(BT * 4 * H);
        lb.rmask = cv.take<float>(B * H);
      }
      h->z = cv.take<float>(B * 4 * H);
      h->zh = gru ? cv.take<float>(B * 3 * H) : nullptr;
      h->hm = cv.take<float>(B * H);
      h->preds = cv.take<float>(BT * O);
      h->var = c.uq ? cv.take<float>(BT * O) : nullptr;
      h->apre = (c.uq && !c.forward_only) ? cv.take<float>(BT * O) : nullptr;
      if (!c.forward_only) {
        h->dz = cv.take<float>(BT * 4 * H);
        h->dz2 = gru ? cv.take<float>(BT * 3 * H) : nullptr;
        h->dy = cv.take<float>(BT * H);
        h->dh_out = cv.take<float>(BT * H);
        h->hp = cv.take<float>(BT * H);
        h->dh_rec = cv.take<float>(B * H);
        h->dc = cv.take<float>(B * H);
        h->dpred = cv.take<float>(BT * O);
        h->da = c.uq ? cv.take<float>(BT * O) : nullptr;
      }
      break;
    case Path::Cluster:
      lfmq::tc_layout(h->tc, c, cv);
      break;
    case Path::General:
      lfmq::gen_layout(h->tc, c, pl, cv);
      break;
    case Path::Dense:
      if (!c.forward_only) {
        h->preds = cv.take<float>(B * O);
        h->dpred = cv.take<float>(B * O);
        h->wpart = cv.take<float>(lfmq::dense_wgrad_scratch(c.max_batch, T * c.n_inputs, O));
      }
      break;
  }
  return cv.off;
}

int validate_dense(const lfmq_dense_config* c) {
  if (!c || c->struct_size != (int32_t)sizeof(lfmq_dense_config)) {
    LFMQ_SET_ERR("lfmq_dense_config: struct_size mismatch (got %d, want %zu)", c ? c->struct_size : -1,
                 sizeof(lfmq_dense_config));
    return LFMQ_ERR_ARG;
  }
  if (c->max_batch <= 0 || c->seq_len <= 0 || c->n_inputs <= 0 || c->n_outputs <= 0) {
    LFMQ_SET_ERR("lfmq_dense_config: non-positive dimension");
    return LFMQ_ERR_ARG;
  }
  if ((int64_t)c->seq_len * c->n_inputs > 48 * 1024) {
    LFMQ_SET_ERR("lfmq_dense_config: seq_len * n_inputs = %lld exceeds %d", (long long)c->seq_len * c->n_inputs,
                 48 * 1024);
    return LFMQ_ERR_UNSUPPORTED;
  }
  if (c->target_idx < 0 || c->target_idx >= c->n_outputs) {
    LFMQ_SET_ERR("lfmq_dense_config: target_idx %d outside [0,%d)", c->target_idx, c->n_outputs);
    return LFMQ_ERR_ARG;
  }
  if (c->optimizer < 0 || c->optimizer > 3) {
    LFMQ_SET_ERR("lfmq_dense_config: unknown optimizer %d", c->optimizer);
    return LFMQ_ERR_ARG;
  }
  if (c->huber_loss && !(c->huber_delta > 0.f)) {
    LFMQ_SET_ERR("lfmq_dense_config: huber_delta must be positive (got %g)", c->huber_delta);
    return LFMQ_ERR_ARG;
  }
  if (c->precision == LFMQ_PREC_BF16 || c->precision == LFMQ_PREC_BF16X3 || c->precision == LFMQ_PREC_TF32) {
    LFMQ_SET_ERR("lfmq_dense_config: the linear model runs in fp32 only: it reads each input once for n_outputs "
                 "multiply-adds, so it is bound by memory bandwidth and tensor cores would not make it faster; "
                 "use LFMQ_PREC_FP32");
    return LFMQ_ERR_UNSUPPORTED;
  }
  if (c->precision != LFMQ_PREC_FP32) {
    LFMQ_SET_ERR("lfmq_dense_config: unknown precision %d", c->precision);
    return LFMQ_ERR_ARG;
  }
  return LFMQ_OK;
}

// Entry points that serve recurrent handles only.
int refuse_dense(lfmq_handle h, const char* fn) {
  if (h && h->path == Path::Dense) {
    LFMQ_SET_ERR("%s: not defined for a dense handle (lfmq_dense_create)", fn);
    return LFMQ_ERR_ARG;
  }
  return 0;
}

#define RUN(expr)                 \
  do {                            \
    int _rc = (expr);             \
    if (_rc != 0) return _rc;     \
  } while (0)

int check_batch(lfmq_handle h, int32_t B) {
  if (!h) {
    LFMQ_SET_ERR("null handle");
    return LFMQ_ERR_ARG;
  }
  if (B <= 0 || B > h->cfg.max_batch) {
    LFMQ_SET_ERR("batch %d outside (0, max_batch=%d]", B, h->cfg.max_batch);
    return LFMQ_ERR_ARG;
  }
  return 0;
}

// Every GEMM of the fp32 step: the fp32 SIMT sgemm, or on a LFMQ_PREC_TF32 handle the same product on wgmma with tf32
// operands (tf32_gemm.cu).  Everything else in forward_fp32 / backward_fp32 is shared by both precisions.
int gemm(lfmq_handle h, cudaStream_t s, int M, int N, int K, const float* A, long sAm, long sAk, const float* B, long sBk,
         long sBn, float* C, long ldc, float beta, float* scratch, size_t scratch_elems) {
  return (h->cfg.precision == LFMQ_PREC_TF32 ? tf32_gemm : sgemm)(s, M, N, K, A, sAm, sAk, B, sBk, sBn, C, ldc, beta,
                                                                  scratch, scratch_elems);
}

// fp32 SIMT (or tf32 GEMM) forward of all layers; fills layers[l].{h,c,y,(gates)} and `preds`.
// uq handles also fill `var` [B,T,O] (and keep the variance head's pre-activation when a backward pass can follow).
// dropout_off: every dropout off, also on a uq handle (training-window attributions only; no entry point of the
// model's own forward sets it).
int forward_fp32(lfmq_handle h, const float* x, int B, int64_t row0, int64_t step, float* preds, float* var,
                 cudaStream_t s, bool dropout_off = false) {
  const lfmq_config& c = h->cfg;
  const int H = c.num_hidden, T = c.seq_len, O = c.n_outputs, L = c.num_layers;
  const float* P = h->params;
  h->prof.begin(LFMQ_REGION_FWD, s);
  for (int l = 0; l < L; ++l) {
    LayerBuf& lb = h->layers[l];
    const lfmq::ParamLayout::Layer& o = h->pl.layers[l];
    const float* in = (l == 0) ? x : h->layers[l - 1].y;
    const int I = o.I;
    const float* rmask = nullptr;
    const bool stochastic = (c.train || c.uq) && !dropout_off;   // rnn_uq_range_estimate.py:86,88: training=True
    if (stochastic && c.recurrent_dropout > 0.f) {
      RUN(gen_row_mask(s, B, H, dropout_key(c.seed, h->tc.stream_base + 2 * l + 1, step, c.recurrent_dropout), row0,
                       lb.rmask));
      rmask = lb.rmask;
    }
    for (int t = 0; t < T && c.rnn_cell == LFMQ_CELL_GRU; ++t) {
      RUN(gemm(h, s, B, 3 * H, I, in + (long)t * I, (long)T * I, 1, P + o.oW, 3 * H, 1, h->z, 3 * H, 0.f, nullptr, 0));
      if (t > 0) {
        const float* hp = rmask ? h->hm : lb.h + (long)(t - 1) * H;
        const long ld = rmask ? H : (long)T * H;
        RUN(gemm(h, s, B, 3 * H, H, hp, ld, 1, P + o.oU, 3 * H, 1, h->zh, 3 * H, 0.f, nullptr, 0));
      }
      RUN(gru_pointwise_fwd(s, B, T, H, t, h->z, t > 0 ? h->zh : nullptr, P + o.ob, lb.gates, lb.h, rmask,
                            rmask ? h->hm : nullptr));
    }
    for (int t = 0; t < T && c.rnn_cell == LFMQ_CELL_LSTM; ++t) {
      RUN(gemm(h, s, B, 4 * H, I, in + (long)t * I, (long)T * I, 1, P + o.oW, 4 * H, 1, h->z, 4 * H, 0.f, nullptr, 0));
      if (t > 0) {
        const float* hp = rmask ? h->hm : lb.h + (long)(t - 1) * H;
        const long ld = rmask ? H : (long)T * H;
        RUN(gemm(h, s, B, 4 * H, H, hp, ld, 1, P + o.oU, 4 * H, 1, h->z, 4 * H, 1.f, nullptr, 0));
      }
      RUN(lstm_pointwise_fwd(s, B, T, H, t, h->z, P + o.ob, lb.gates, lb.c, lb.h, rmask, rmask ? h->hm : nullptr));
    }
    const bool drop = stochastic && c.dropout > 0.f;
    RUN(bn_dropout_fwd(s, B, T, H, lb.h, P + o.ogamma, P + o.obeta, P + o.omean, P + o.ovar, c.bn_epsilon, drop,
                       dropout_key(c.seed, h->tc.stream_base + 2 * l, step, c.dropout), row0, lb.y));
  }
  h->prof.end(LFMQ_REGION_FWD, s);
  h->prof.begin(LFMQ_REGION_HEAD, s);
  const float* yl = h->layers[L - 1].y;
  RUN(gemm(h, s, B * T, O, H, yl, H, 1, P + h->pl.oWo, O, 1, preds, O, 0.f, nullptr, 0));
  RUN(add_bias_rows(s, (long)B * T, O, preds, P + h->pl.obo));
  if (c.uq) {
    float* a = h->apre ? h->apre : var;           // forward-only handles activate in place
    RUN(gemm(h, s, B * T, O, H, yl, H, 1, P + h->pl.oWv, O, 1, a, O, 0.f, nullptr, 0));
    RUN(add_bias_rows(s, (long)B * T, O, a, P + h->pl.obv));
    RUN(softplus_floor(s, (long)B * T * O, a, var));
  }
  h->prof.end(LFMQ_REGION_HEAD, s);
  return 0;
}

// dx_out (nullable): dLoss/dx [B,T,F] of the lowest layer (the stages of a forecast chain feed predictions back in).
// input_only: the dz / dh chain and the dx GEMMs alone, for integrated gradients: no parameter gradient (head, BN, dW,
// dU, db) is formed, and the handle's gradient buffer is not written.
int backward_fp32(lfmq_handle h, const float* x, int B, cudaStream_t s, float* dx_out = nullptr,
                  bool input_only = false) {
  const lfmq_config& c = h->cfg;
  const int H = c.num_hidden, T = c.seq_len, O = c.n_outputs, L = c.num_layers;
  const long BT = (long)B * T;
  const float* P = h->params;
  float* G = h->grads;
  const float* yl = h->layers[L - 1].y;
  // head: dWo = y^T dpred, dbo = colsum(dpred), dy = dpred Wo^T
  h->prof.begin(LFMQ_REGION_HEAD, s);
  if (!input_only) {
    RUN(gemm(h, s, H, O, (int)BT, yl, 1, H, h->dpred, O, 1, G + h->pl.oWo, O, 0.f, h->scratch, h->scratch_elems));
    RUN(colsum(s, BT, O, h->dpred, G + h->pl.obo, h->scratch, h->scratch_elems));
  }
  RUN(gemm(h, s, (int)BT, H, O, h->dpred, O, 1, P + h->pl.oWo, 1, O, h->dy, H, 0.f, nullptr, 0));
  if (c.uq) {      // variance head: same three products on da, dy accumulates
    if (!input_only) {
      RUN(gemm(h, s, H, O, (int)BT, yl, 1, H, h->da, O, 1, G + h->pl.oWv, O, 0.f, h->scratch, h->scratch_elems));
      RUN(colsum(s, BT, O, h->da, G + h->pl.obv, h->scratch, h->scratch_elems));
    }
    RUN(gemm(h, s, (int)BT, H, O, h->da, O, 1, P + h->pl.oWv, 1, O, h->dy, H, 1.f, nullptr, 0));
  }
  h->prof.end(LFMQ_REGION_HEAD, s);
  for (int l = L - 1; l >= 0; --l) {
    LayerBuf& lb = h->layers[l];
    const lfmq::ParamLayout::Layer& o = h->pl.layers[l];
    const int I = o.I;
    const float* rmask = ((c.train || c.uq) && c.recurrent_dropout > 0.f) ? lb.rmask : nullptr;
    const bool drop = (c.train || c.uq) && c.dropout > 0.f;
    h->prof.begin(LFMQ_REGION_BWD, s);
    RUN(bn_dropout_bwd(s, B, T, H, h->dy, lb.h, P + o.ogamma, P + o.omean, P + o.ovar, c.bn_epsilon, drop,
                       dropout_key(c.seed, h->tc.stream_base + 2 * l, h->last_step, c.dropout), h->last_row0, h->dh_out,
                       input_only ? nullptr : G + o.ogamma, input_only ? nullptr : G + o.obeta, h->scratch,
                       h->scratch_elems));
    const bool gru = c.rnn_cell == LFMQ_CELL_GRU;
    const int NG = gru ? 3 : 4;
    for (int t = T - 1; t >= 0 && gru; --t) {
      RUN(gru_pointwise_bwd(s, B, T, H, t, lb.gates, lb.h, h->dh_out, (t < T - 1) ? h->dh_rec : nullptr, rmask, h->dc,
                            h->dz, h->dz2));
      if (t > 0)
        RUN(gemm(h, s, B, H, 3 * H, h->dz2 + (long)t * 3 * H, (long)T * 3 * H, 1, P + o.oU, 1, 3 * H, h->dh_rec, H, 0.f,
                  nullptr, 0));
    }
    for (int t = T - 1; t >= 0 && !gru; --t) {
      RUN(lstm_pointwise_bwd(s, B, T, H, t, lb.gates, lb.c, h->dh_out, (t < T - 1) ? h->dh_rec : nullptr, rmask, h->dc,
                             h->dz));
      if (t > 0)
        RUN(gemm(h, s, B, H, 4 * H, h->dz + (long)t * 4 * H, (long)T * 4 * H, 1, P + o.oU, 1, 4 * H, h->dh_rec, H, 0.f,
                  nullptr, 0));
    }
    h->prof.end(LFMQ_REGION_BWD, s);
    h->prof.begin(LFMQ_REGION_WGRAD, s);
    const float* in = (l == 0) ? x : h->layers[l - 1].y;
    // LSTM: one gradient buffer feeds dW, dU and db.  GRU: dz = d(input projection), dz2 = d(recurrent projection),
    // bias rows [2][3H] = colsum of each.
    const float* dzr = gru ? h->dz2 : h->dz;
    const int GH = NG * H;
    if (!input_only) {
      RUN(gemm(h, s, I, GH, (int)BT, in, 1, I, h->dz, GH, 1, G + o.oW, GH, 0.f, h->scratch, h->scratch_elems));
      RUN(shift_mask(s, B, T, H, lb.h, rmask, h->hp));
      RUN(gemm(h, s, H, GH, (int)BT, h->hp, 1, H, dzr, GH, 1, G + o.oU, GH, 0.f, h->scratch, h->scratch_elems));
      RUN(colsum(s, BT, GH, h->dz, G + o.ob, h->scratch, h->scratch_elems));
      if (gru) RUN(colsum(s, BT, GH, h->dz2, G + o.ob + GH, h->scratch, h->scratch_elems));
    }
    if (l > 0 || dx_out)
      RUN(gemm(h, s, (int)BT, I, GH, h->dz, GH, 1, P + o.oW, 1, GH, l > 0 ? h->dy : dx_out, I, 0.f, nullptr, 0));
    h->prof.end(LFMQ_REGION_WGRAD, s);
  }
  return 0;
}

// optimizer update with the clip scale already in the gradient tail (LFMQ_TAIL_CLIP_SCALE) + the MaxNorm kernel
// constraint
int apply_update(lfmq_handle h, float lr, int64_t iteration, cudaStream_t s) {
  const lfmq_config& c = h->cfg;
  float* tail = h->grads + h->n_train;
  float lr_eff = lr;
  if (c.optimizer == LFMQ_OPT_ADAM) {
    const double t = (double)(iteration + 1);
    lr_eff = (float)((double)lr * sqrt(1.0 - pow(0.999, t)) / (1.0 - pow(0.9, t)));
  }
  RUN(opt_update(s, c.optimizer, h->n_train, h->params, h->grads, h->slots,
                 h->n_slots > 1 ? h->slots + h->n_train : nullptr, tail + LFMQ_TAIL_GRAD_NORM, lr_eff, 0.f, 0.f,
                 c.sgd_momentum));
  for (const lfmq::ParamLayout::Layer& o : h->pl.layers)
    RUN(maxnorm_cols(s, o.I, (c.rnn_cell == LFMQ_CELL_GRU ? 3 : 4) * c.num_hidden, h->params + o.oW, c.max_norm));
  h->tc.weights_dirty = 1;
  return 0;
}

// ---- a model is a chain of S >= 1 stages; a single handle is the chain of one stage with weight 1 ----------------
// None of these touch tc.stream_base: only the public chain entry points (chain_check) number the stages' dropout
// streams, so a handle that is stage s > 0 of a chain keeps its streams when it is called on its own.

// The forward of every stage in order.  Stage i > 0 reads the window built in work slot i - 1 from stage i - 1's target
// predictions (rnn_uq_range_estimate.py:118: outputs[-2]; variances never feed forward); one stage needs no work.
// preds == nullptr is the training path: forward_fp32 into each handle's own preds / var, which the backward reads.
// Otherwise the predict path: preds[i] (and vars[i] on a uq chain) through lfmq_forward / lfmq_forward_uq, which
// dispatch on the stage's precision.
int run_stages(const lfmq_handle* st, int S, const float* x, int B, int64_t row0, int64_t step, float* const* preds,
               float* const* vars, float* work, cudaStream_t s) {
  const lfmq_config& c = st[0]->cfg;
  const size_t slot = (size_t)B * c.seq_len * c.n_inputs;
  const float* in = x;
  for (int i = 0; i < S; ++i) {
    lfmq_handle h = st[i];
    if (i > 0) {
      float* next = work + (size_t)(i - 1) * slot;
      RUN(chain_next_input(s, B, c.seq_len, c.n_inputs, c.n_outputs, in, preds ? preds[i - 1] : st[i - 1]->preds, x,
                           next));
      in = next;
    }
    if (preds && c.uq) {
      RUN(lfmq_forward_uq(h, in, B, row0, step, preds[i], vars[i], s));
    } else if (preds) {
      RUN(lfmq_forward(h, in, B, row0, step, preds[i], s));
    } else {
      h->last_step = step;
      h->last_row0 = row0;
      RUN(forward_fp32(h, in, B, row0, step, h->preds, h->var, s));
    }
  }
  return 0;
}

// Every stage's {B, unmasked rows, unmasked last-step rows} into out_dev[3 * i], in one loss pass without predictions;
// their weighted sums for a stage with row weights.
int stage_counts(const lfmq_handle* st, int S, const float* const* y, int B, float* out_dev, cudaStream_t s) {
  lfmq::ChainUqArgs a{};
  for (int i = 0; i < S; ++i) {
    a.y.p[i] = const_cast<float*>(y[i]);
    a.counts.p[i] = out_dev + 3 * i;
    a.rw.p[i] = st[i]->tc.row_w;
  }
  const lfmq_config& c = st[0]->cfg;
  return chain_uq_loss_grad(s, S, B, c.seq_len, c.n_outputs, a, c.target_idx, c.target_lambda, c.rnn_lambda, nullptr,
                            st[0]->scratch);
}

// A point handle's own batch counts into h->sc->denom: {B, unmasked rows}, or with row weights {sum of weights,
// weighted unmasked rows} (and a third count), from the weighted count pass of stage_counts.
int point_counts(lfmq_handle h, const float* y, int B, cudaStream_t s) {
  if (h->tc.row_w) return stage_counts(&h, 1, &y, B, h->sc->denom, s);
  return mask_count(s, B, h->cfg.seq_len, h->cfg.n_outputs, y, h->sc->denom, h->sc->mask_tickets);
}

// The uq loss of the stages' own preds / var (train.py:201-218): one loss pass over all stages for the mask counts
// unless denom brings them, and one for the losses and w_s * dLoss_s / d(pred_s, variance pre-activation_s).
int stages_loss_uq(const lfmq_handle* st, int S, const float* const* y, const float* weights, int B, const float* denom,
                   float* loss_out_dev, cudaStream_t s) {
  const lfmq_config& c0 = st[0]->cfg;
  const int T = c0.seq_len, O = c0.n_outputs;
  lfmq::ChainUqArgs a{};
  for (int i = 0; i < S; ++i) {
    a.y.p[i] = const_cast<float*>(y[i]);
    a.counts.p[i] = denom ? const_cast<float*>(denom) + 3 * i : st[i]->sc->denom;
    a.rw.p[i] = st[i]->tc.row_w;
    a.w.w[i] = weights[i];
  }
  float* scratch = st[0]->scratch;
  if (!denom) RUN(chain_uq_loss_grad(s, S, B, T, O, a, c0.target_idx, c0.target_lambda, c0.rnn_lambda, nullptr, scratch));
  for (int i = 0; i < S; ++i) {
    a.pred.p[i] = st[i]->preds;
    a.var.p[i] = st[i]->var;
    a.apre.p[i] = st[i]->apre;
    a.dpred.p[i] = st[i]->dpred;
    a.da.p[i] = st[i]->da;
    float* tail = st[i]->grads + st[i]->n_train;
    a.loss.p[i] = tail + LFMQ_TAIL_LOSS;
    a.mse0.p[i] = tail + LFMQ_TAIL_MSE0;
    a.uq0.p[i] = tail + LFMQ_TAIL_UQ_LOSS_LAST_TAR;
  }
  a.counts_in = 1;
  return chain_uq_loss_grad(s, S, B, T, O, a, c0.target_idx, c0.target_lambda, c0.rnn_lambda, loss_out_dev, scratch);
}

// Forward, loss and BPTT of S training-mode fp32 stages of one kind: the body of lfmq_backward's fp32 branches and of
// lfmq_chain_backward(_dp).  denom (nullable): three counts per stage, summed over the data-parallel ranks; a point
// stage reads the two that lead them, {B, mask_count}.  Without it every stage counts its own batch.
// loss_out_dev (nullable): the weighted sums over the stages.  work is read only when S > 1.
int backward_stages(const lfmq_handle* st, int S, const float* x, const float* const* y, const float* weights, int B,
                    int64_t row0, int64_t step, const float* denom, float* work, float* loss_out_dev, cudaStream_t s) {
  const lfmq_config& c0 = st[0]->cfg;
  const int T = c0.seq_len, F = c0.n_inputs, O = c0.n_outputs;
  const size_t slot = (size_t)B * T * F;
  // forward of every stage (each keeps its own saved state), then each stage's loss and dLoss/dpred_s, weighted
  RUN(run_stages(st, S, x, B, row0, step, nullptr, nullptr, work, s));
  lfmq::ChainPtrs dpred{}, l2{}, none{};
  lfmq::ChainWeights w{};
  if (c0.uq) RUN(stages_loss_uq(st, S, y, weights, B, denom, loss_out_dev, s));
  for (int i = 0; i < S && !c0.uq; ++i) {
    lfmq_handle h = st[i];
    const lfmq_config& c = h->cfg;
    const float* d = denom ? denom + 3 * i : h->sc->denom;
    if (!denom) RUN(point_counts(h, y[i], B, s));
    float* tail = h->grads + h->n_train;
    RUN(loss_grad(s, B, T, O, h->preds, y[i], d, h->tc.row_w, c.target_idx, c.target_lambda, c.rnn_lambda, h->dpred,
                  tail, nullptr, h->scratch));
    if (weights[i] != 1.0f) RUN(scale_inplace(s, (long)B * T * O, h->dpred, weights[i]));
    l2.p[i] = tail;
    w.w[i] = weights[i];
  }
  if (loss_out_dev && !c0.uq) RUN(chain_combine(s, S, none, 0.f, l2, w, loss_out_dev));
  // BPTT from the last stage down; the input gradient of stage i lands on the last time step of earlier predictions
  // (the target predictions on a uq chain: variances never feed forward, so there is no dvar feedback)
  for (int i = 0; i < S; ++i) dpred.p[i] = st[i]->dpred;
  for (int i = S - 1; i >= 1; --i) {
    float* dx = work + (size_t)(S - 1) * slot;
    const float* in_i = work + (size_t)(i - 1) * slot;
    RUN(backward_fp32(st[i], in_i, B, s, dx));
    RUN(chain_scatter_dx(s, B, T, F, O, i, dx, dpred));
  }
  return backward_fp32(st[0], x, B, s);
}

// The analyses carve the caller's work on 256-byte granules of the work pointer, with one layout function each: run on
// base == nullptr it gives the size their *_work_bytes report, run on work it gives the buffers.
constexpr size_t kWorkGranule = 256;

template <typename Layout>
size_t work_size(const Layout& layout) {
  Carver cv{nullptr, 0, kWorkGranule};
  layout(cv);
  return cv.off;
}

template <typename Layout>
int32_t report_work_bytes(uint64_t* bytes, const char* fn, const Layout& layout) {
  if (!bytes) {
    LFMQ_SET_ERR("%s: bytes == NULL", fn);
    return LFMQ_ERR_ARG;
  }
  *bytes = work_size(layout);
  return LFMQ_OK;
}

// *out = the buffers `layout` carves from work, which must hold all of them
template <typename Layout, typename Work>
int carve_work(void* work, uint64_t work_bytes, const char* fn, const Layout& layout, Work* out) {
  const size_t need = work_size(layout);
  if (!work || work_bytes < need) {
    LFMQ_SET_ERR("%s: work needs %zu bytes, got %llu", fn, need, (unsigned long long)work_bytes);
    return LFMQ_ERR_WORKSPACE;
  }
  Carver cv{static_cast<char*>(work), 0, kWorkGranule};
  *out = layout(cv);
  return 0;
}
}  // namespace

// =============================================================================================
extern "C" {

const char* lfmq_last_error(void) { return lfmq::g_err; }
int32_t lfmq_abi_version(void) { return LFMQ_ABI_VERSION; }
int64_t lfmq_launch_count(void) { return lfmq::g_launches; }

namespace {
void dense_handle_config(const lfmq_dense_config* d, lfmq_handle_s* h) {
  lfmq_config& c = h->cfg;
  memset(&c, 0, sizeof(c));
  c.struct_size = (int32_t)sizeof(lfmq_config);
  c.max_batch = d->max_batch;
  c.seq_len = d->seq_len;
  c.n_inputs = d->n_inputs;
  c.n_outputs = d->n_outputs;
  c.target_idx = d->target_idx;
  c.precision = d->precision;
  c.optimizer = d->optimizer;
  c.forward_only = d->forward_only;
  c.target_lambda = d->target_lambda;
  c.max_grad_norm = d->max_grad_norm;
  c.sgd_momentum = d->sgd_momentum;
  h->path = Path::Dense;
  h->huber = d->huber_loss ? 1 : 0;
  h->huber_delta = d->huber_delta;
}

// The body of lfmq_workspace_bytes and lfmq_dense_workspace_bytes
int32_t workspace_bytes_of(lfmq_handle_s& h, bool with_path, uint64_t* bytes) {
  if (!bytes) {
    LFMQ_SET_ERR("bytes == NULL");
    return LFMQ_ERR_ARG;
  }
  *bytes = layout(&h, nullptr, with_path) + WS_ALIGN;
  return LFMQ_OK;
}

// The body of lfmq_create and lfmq_dense_create.  h carries its config and path; path_rc is choose_path's result (its
// message still in g_err), reported once the workspace is large enough for what lfmq_workspace_bytes sized.
int32_t create(std::unique_ptr<lfmq_handle_s> h, int path_rc, void* workspace, uint64_t workspace_bytes,
               lfmq_handle* out) {
  if (!workspace || !out) {
    LFMQ_SET_ERR("workspace/out == NULL");
    return LFMQ_ERR_ARG;
  }
  char* base = reinterpret_cast<char*>(ws_align_up(reinterpret_cast<size_t>(workspace)));
  const size_t need = layout(h.get(), nullptr, path_rc == 0) + (base - reinterpret_cast<char*>(workspace));
  if (need > workspace_bytes) {
    LFMQ_SET_ERR("workspace too small: need %zu bytes, got %llu", need, (unsigned long long)workspace_bytes);
    return LFMQ_ERR_WORKSPACE;
  }
  RUN(path_rc);
  layout(h.get(), base, true);
  h->tc.prof = &h->prof;
  if (h->path == Path::Cluster) RUN(lfmq::tc_init(h->tc, h->cfg));
  if (h->path == Path::General) RUN(lfmq::gen_init(h->tc, h->cfg));
  // zero parameters / gradients / optimizer slots / scalars; BN moving_variance = 1
  LFMQ_CUDA_CHECK(cudaMemsetAsync(h->params, 0, sizeof(float) * h->n_total, 0));
  LFMQ_CUDA_CHECK(cudaMemsetAsync(h->grads, 0, sizeof(float) * h->n_grad_buf, 0));
  if (h->slots) LFMQ_CUDA_CHECK(cudaMemsetAsync(h->slots, 0, sizeof(float) * h->n_slots * h->n_train, 0));
  LFMQ_CUDA_CHECK(cudaMemsetAsync(h->sc, 0, sizeof(Scalars), 0));
  for (const lfmq::ParamLayout::Layer& o : h->pl.layers)
    RUN(lfmq::fill(0, h->params + o.ovar, h->cfg.num_hidden, 1.0f));
  LFMQ_CUDA_CHECK(cudaStreamSynchronize(0));
  *out = h.release();
  return LFMQ_OK;
}
}  // namespace

int32_t lfmq_workspace_bytes(const lfmq_config* cfg, uint64_t* bytes) {
  RUN(validate(cfg));
  lfmq_handle_s h;
  h.cfg = *cfg;
  const bool supported = choose_path(h.cfg, &h.path) == 0;     // lfmq_create reports an unsupported configuration
  return workspace_bytes_of(h, supported, bytes);
}

int32_t lfmq_create(const lfmq_config* cfg, void* workspace, uint64_t workspace_bytes, lfmq_handle* out) {
  RUN(validate(cfg));
  auto h = std::make_unique<lfmq_handle_s>();
  h->cfg = *cfg;
  const int path_rc = choose_path(h->cfg, &h->path);
  return create(std::move(h), path_rc, workspace, workspace_bytes, out);
}

int32_t lfmq_dense_workspace_bytes(const lfmq_dense_config* cfg, uint64_t* bytes) {
  RUN(validate_dense(cfg));
  lfmq_handle_s h;
  dense_handle_config(cfg, &h);
  return workspace_bytes_of(h, true, bytes);
}

int32_t lfmq_dense_create(const lfmq_dense_config* cfg, void* workspace, uint64_t workspace_bytes, lfmq_handle* out) {
  RUN(validate_dense(cfg));
  auto h = std::make_unique<lfmq_handle_s>();
  dense_handle_config(cfg, h.get());
  return create(std::move(h), 0, workspace, workspace_bytes, out);
}

int32_t lfmq_destroy(lfmq_handle h) {
  delete h;
  return LFMQ_OK;
}

int32_t lfmq_param_count(lfmq_handle h, int32_t* n_tensors, int64_t* n_trainable, int64_t* n_total) {
  if (!h) {
    LFMQ_SET_ERR("null handle");
    return LFMQ_ERR_ARG;
  }
  if (n_tensors) *n_tensors = (int32_t)h->specs.size();
  if (n_trainable) *n_trainable = h->n_train;
  if (n_total) *n_total = h->n_total;
  return LFMQ_OK;
}

int32_t lfmq_param_spec(lfmq_handle h, int32_t index, char* name, int32_t name_cap, int32_t* ndim, int64_t shape[2],
                        int64_t* offset_elems, int32_t* trainable) {
  if (!h || index < 0 || index >= (int32_t)h->specs.size()) {
    LFMQ_SET_ERR("lfmq_param_spec: bad handle or index %d", index);
    return LFMQ_ERR_ARG;
  }
  const ParamSpec& p = h->specs[index];
  if (name && name_cap > 0) {
    strncpy(name, p.name.c_str(), name_cap - 1);
    name[name_cap - 1] = 0;
  }
  if (ndim) *ndim = p.ndim;
  if (shape) {
    shape[0] = p.shape[0];
    shape[1] = p.shape[1];
  }
  if (offset_elems) *offset_elems = p.offset;
  if (trainable) *trainable = p.trainable;
  return LFMQ_OK;
}

int32_t lfmq_set_device_share(lfmq_handle h, int32_t num, int32_t den) {
  if (!h || num < 1 || den < num) {
    LFMQ_SET_ERR("lfmq_set_device_share: need a handle and 0 < num <= den (got %d/%d)", num, den);
    return LFMQ_ERR_ARG;
  }
  h->tc.share_num = num;
  h->tc.share_den = den;
  return LFMQ_OK;
}

int32_t lfmq_persistent_cta_budget(int32_t sm_count, int32_t ctas_per_sm, int32_t num, int32_t den, int64_t* budget) {
  if (sm_count < 1 || ctas_per_sm < 1 || num < 1 || den < num || !budget) {
    LFMQ_SET_ERR("lfmq_persistent_cta_budget: need sm_count, ctas_per_sm >= 1 and 0 < num <= den (got %d, %d, %d/%d)",
                 sm_count, ctas_per_sm, num, den);
    return LFMQ_ERR_ARG;
  }
  *budget = lfmq::persistent_cta_budget(sm_count, ctas_per_sm, num, den);
  return LFMQ_OK;
}

int32_t lfmq_params_ptr(lfmq_handle h, float** dev) {
  if (!h || !dev) return LFMQ_ERR_ARG;
  *dev = h->params;
  return LFMQ_OK;
}
int32_t lfmq_grads_ptr(lfmq_handle h, float** dev) {
  if (!h || !dev) return LFMQ_ERR_ARG;
  *dev = h->grads;
  return LFMQ_OK;
}
int32_t lfmq_opt_state_ptr(lfmq_handle h, float** dev, int64_t* n_elems) {
  if (!h || !dev) return LFMQ_ERR_ARG;
  *dev = h->slots;
  if (n_elems) *n_elems = h->slots ? (int64_t)h->n_slots * h->n_train : 0;
  return LFMQ_OK;
}

int32_t lfmq_set_params(lfmq_handle h, const float* host, int64_t n, void* stream) {
  if (!h || !host || n != h->n_total) {
    LFMQ_SET_ERR("lfmq_set_params: expected %lld elements, got %lld", h ? (long long)h->n_total : -1LL, (long long)n);
    return LFMQ_ERR_ARG;
  }
  LFMQ_CUDA_CHECK(cudaMemcpyAsync(h->params, host, sizeof(float) * n, cudaMemcpyHostToDevice, (cudaStream_t)stream));
  LFMQ_CUDA_CHECK(cudaStreamSynchronize((cudaStream_t)stream));
  h->tc.weights_dirty = 1;
  return LFMQ_OK;
}

int32_t lfmq_get_params(lfmq_handle h, float* host, int64_t n, void* stream) {
  if (!h || !host || n != h->n_total) {
    LFMQ_SET_ERR("lfmq_get_params: expected %lld elements, got %lld", h ? (long long)h->n_total : -1LL, (long long)n);
    return LFMQ_ERR_ARG;
  }
  LFMQ_CUDA_CHECK(cudaMemcpyAsync(host, h->params, sizeof(float) * n, cudaMemcpyDeviceToHost, (cudaStream_t)stream));
  LFMQ_CUDA_CHECK(cudaStreamSynchronize((cudaStream_t)stream));
  return LFMQ_OK;
}

int32_t lfmq_forward(lfmq_handle h, const float* x, int32_t B, int64_t row0, int64_t step, float* preds, void* stream) {
  RUN(check_batch(h, B));
  if (!x || !preds) {
    LFMQ_SET_ERR("lfmq_forward: null pointer");
    return LFMQ_ERR_ARG;
  }
  cudaStream_t s = (cudaStream_t)stream;
  h->last_step = step;
  h->last_row0 = row0;
  if (h->cfg.uq) {
    LFMQ_SET_ERR("lfmq_forward: uq handle, call lfmq_forward_uq");
    return LFMQ_ERR_ARG;
  }
  const lfmq_config& c = h->cfg;
  switch (h->path) {
    case Path::Fp32:
      return forward_fp32(h, x, B, row0, step, preds, nullptr, s);
    case Path::Cluster:
      return lfmq::tc_forward(h->tc, c, h->pl, h->params, x, B, row0, step, preds, /*save=*/false, s);
    case Path::General:
      return lfmq::gen_forward(h->tc, c, h->pl, h->params, x, B, row0, step, preds, s);
    case Path::Dense:
      break;
  }
  h->prof.begin(LFMQ_REGION_FWD, s);
  RUN(dense_forward(s, x, B, c.seq_len * c.n_inputs, c.n_outputs, h->params + h->pl.oWo, h->params + h->pl.obo, preds));
  h->prof.end(LFMQ_REGION_FWD, s);
  return LFMQ_OK;
}

int32_t lfmq_forward_uq(lfmq_handle h, const float* x, int32_t B, int64_t row0, int64_t step, float* preds, float* var,
                        void* stream) {
  RUN(check_batch(h, B));
  if (!x || !preds || !var) {
    LFMQ_SET_ERR("lfmq_forward_uq: null pointer");
    return LFMQ_ERR_ARG;
  }
  if (!h->cfg.uq) {
    LFMQ_SET_ERR("lfmq_forward_uq: handle was created with uq = 0");
    return LFMQ_ERR_ARG;
  }
  h->last_step = step;
  h->last_row0 = row0;
  if (h->path == Path::General)      // a uq handle runs the fp32 step or the general path
    return lfmq::gen_forward_uq(h->tc, h->cfg, h->pl, h->params, x, B, row0, step, preds, var, (cudaStream_t)stream);
  return forward_fp32(h, x, B, row0, step, preds, var, (cudaStream_t)stream);
}

int32_t lfmq_loss(lfmq_handle h, const float* preds, const float* y, int32_t B, float* out_dev, void* stream) {
  // validation stacks every batch (train.py:318-329), so B may exceed max_batch here: the loss needs no workspace
  if (!h || B <= 0) {
    LFMQ_SET_ERR("lfmq_loss: bad handle or batch %d", B);
    return LFMQ_ERR_ARG;
  }
  if (!preds || !y || !out_dev) {
    LFMQ_SET_ERR("lfmq_loss: null pointer");
    return LFMQ_ERR_ARG;
  }
  const lfmq_config& c = h->cfg;
  if (h->path == Path::Dense)    // validation: the MSE form whatever huber_loss is (losses.py:102, is_validation=True)
    return dense_loss((cudaStream_t)stream, preds, y, B, c.n_outputs, nullptr, nullptr, c.target_idx, c.target_lambda, 0,
                      1.f, nullptr, out_dev, h->scratch);
  return loss_grad((cudaStream_t)stream, B, c.seq_len, c.n_outputs, preds, y, nullptr, nullptr, c.target_idx,
                   c.target_lambda, c.rnn_lambda, nullptr, out_dev, nullptr, h->scratch);
}

int32_t lfmq_loss_uq(lfmq_handle h, const float* preds, const float* var, const float* y, int32_t B, float* out_dev,
                     void* stream) {
  if (!h || B <= 0 || !preds || !var || !y || !out_dev) {
    LFMQ_SET_ERR("lfmq_loss_uq: bad handle, batch %d or null pointer", B);
    return LFMQ_ERR_ARG;
  }
  RUN(refuse_dense(h, "lfmq_loss_uq"));
  const lfmq_config& c = h->cfg;
  lfmq::ChainUqArgs a{};      // one stage of weight 1: the weighted sums {uq_loss, uq_loss_last_tar, mse} are its own
  a.pred.p[0] = const_cast<float*>(preds);
  a.var.p[0] = const_cast<float*>(var);
  a.y.p[0] = const_cast<float*>(y);
  a.w.w[0] = 1.0f;
  return chain_uq_loss_grad((cudaStream_t)stream, 1, B, c.seq_len, c.n_outputs, a, c.target_idx, c.target_lambda,
                            c.rnn_lambda, out_dev, h->scratch);
}

int32_t lfmq_mask_count(lfmq_handle h, const float* y, int32_t B, float* out_dev, void* stream) {
  RUN(check_batch(h, B));
  if (!y || !out_dev) {
    LFMQ_SET_ERR("lfmq_mask_count: null pointer");
    return LFMQ_ERR_ARG;
  }
  if (h->path == Path::Dense)
    return dense_loss((cudaStream_t)stream, nullptr, y, B, h->cfg.n_outputs, nullptr, h->tc.row_w, 0, 0.f, 0, 1.f,
                      nullptr, out_dev, h->scratch);
  if (!h->tc.row_w)
    return mask_count((cudaStream_t)stream, B, h->cfg.seq_len, h->cfg.n_outputs, y, out_dev, h->sc->mask_tickets);
  RUN(point_counts(h, y, B, (cudaStream_t)stream));     // three counts: the first two are the caller's
  LFMQ_CUDA_CHECK(cudaMemcpyAsync(out_dev, h->sc->denom, 2 * sizeof(float), cudaMemcpyDeviceToDevice,
                                  (cudaStream_t)stream));
  return LFMQ_OK;
}

int32_t lfmq_mask_count_uq(lfmq_handle h, const float* y, int32_t B, float* out_dev, void* stream) {
  RUN(check_batch(h, B));
  if (!y || !out_dev) {
    LFMQ_SET_ERR("lfmq_mask_count_uq: null pointer");
    return LFMQ_ERR_ARG;
  }
  RUN(refuse_dense(h, "lfmq_mask_count_uq"));
  return stage_counts(&h, 1, &y, B, out_dev, (cudaStream_t)stream);
}

int32_t lfmq_set_row_weights(lfmq_handle h, const float* w_dev) {
  if (!h) {
    LFMQ_SET_ERR("lfmq_set_row_weights: null handle");
    return LFMQ_ERR_ARG;
  }
  if (h->cfg.forward_only) {
    LFMQ_SET_ERR("lfmq_set_row_weights: handle was created forward_only");
    return LFMQ_ERR_UNSUPPORTED;
  }
  h->tc.row_w = w_dev;
  return LFMQ_OK;
}

int32_t lfmq_backward(lfmq_handle h, const float* x, const float* y, int32_t B, int64_t row0, int64_t step,
                      const float* denom_dev, void* stream) {
  RUN(check_batch(h, B));
  if (!x || !y) {
    LFMQ_SET_ERR("lfmq_backward: null pointer");
    return LFMQ_ERR_ARG;
  }
  if (h->cfg.forward_only) {
    LFMQ_SET_ERR("lfmq_backward: handle was created forward_only");
    return LFMQ_ERR_UNSUPPORTED;
  }
  cudaStream_t s = (cudaStream_t)stream;
  const lfmq_config& c = h->cfg;
  float* tail = h->grads + h->n_train;
  switch (h->path) {
    case Path::Fp32: {    // a trainable uq handle always runs this path
      // denom_dev: stage 0's counts, the three of lfmq_mask_count_uq or the two of lfmq_mask_count
      const float one = 1.0f;
      return backward_stages(&h, 1, x, &y, &one, B, row0, step, denom_dev, nullptr, nullptr, s);
    }
    case Path::Cluster:
    case Path::General: {
      const float* denom = denom_dev;
      if (!denom) {
        RUN(point_counts(h, y, B, s));
        denom = h->sc->denom;
      }
      if (h->path == Path::Cluster)
        return lfmq::tc_backward(h->tc, c, h->pl, h->params, h->grads, x, y, B, row0, step, denom, tail, s);
      return lfmq::gen_backward(h->tc, c, h->pl, h->params, h->grads, x, y, B, row0, step, denom, tail, s);
    }
    case Path::Dense:
      break;
  }
  // the dense model: the forward into the handle's own preds, the loss and dLoss/dpred, then dW and db
  const int K = c.seq_len * c.n_inputs, O = c.n_outputs;
  h->prof.begin(LFMQ_REGION_FWD, s);
  RUN(dense_forward(s, x, B, K, O, h->params + h->pl.oWo, h->params + h->pl.obo, h->preds));
  h->prof.end(LFMQ_REGION_FWD, s);
  h->prof.begin(LFMQ_REGION_HEAD, s);
  const float* denom = denom_dev;
  if (!denom && h->tc.row_w) {    // the weighted means divide by the batch's weight sum
    RUN(dense_loss(s, nullptr, y, B, O, nullptr, h->tc.row_w, 0, 0.f, 0, 1.f, nullptr, h->sc->denom, h->scratch));
    denom = h->sc->denom;
  }
  RUN(dense_loss(s, h->preds, y, B, O, denom, h->tc.row_w, c.target_idx, c.target_lambda, h->huber, h->huber_delta,
                 h->dpred, tail, h->scratch));
  h->prof.end(LFMQ_REGION_HEAD, s);
  h->prof.begin(LFMQ_REGION_WGRAD, s);
  RUN(dense_wgrad(s, x, h->dpred, B, K, O, h->wpart, h->grads));
  h->prof.end(LFMQ_REGION_WGRAD, s);
  return LFMQ_OK;
}

int32_t lfmq_apply(lfmq_handle h, float lr, int64_t iteration, void* stream) {
  if (!h || h->cfg.forward_only) {
    LFMQ_SET_ERR("lfmq_apply: bad handle");
    return LFMQ_ERR_ARG;
  }
  cudaStream_t s = (cudaStream_t)stream;
  const lfmq_config& c = h->cfg;
  float* tail = h->grads + h->n_train;
  h->prof.begin(LFMQ_REGION_OPT, s);
  RUN(grad_norm_scale(s, h->n_train, h->grads, c.max_grad_norm, tail + LFMQ_TAIL_GRAD_NORM, h->scratch,
                      &h->sc->norm_ticket));
  RUN(apply_update(h, lr, iteration, s));
  h->prof.end(LFMQ_REGION_OPT, s);
  return LFMQ_OK;
}

int32_t lfmq_train_step(lfmq_handle h, const float* x, const float* y, int32_t B, int64_t row0, int64_t step, float lr,
                        float* loss_out_dev, void* stream) {
  RUN(lfmq_backward(h, x, y, B, row0, step, nullptr, stream));
  RUN(lfmq_apply(h, lr, step, stream));
  const float* tail = h->grads + h->n_train;
  if (loss_out_dev && !h->cfg.uq)      // {loss, mse_0}
    LFMQ_CUDA_CHECK(cudaMemcpyAsync(loss_out_dev, tail + LFMQ_TAIL_LOSS, 2 * sizeof(float), cudaMemcpyDeviceToDevice,
                                    (cudaStream_t)stream));
  if (loss_out_dev && h->cfg.uq) {      // {uq_loss_last_tar, mse_0}
    LFMQ_CUDA_CHECK(cudaMemcpyAsync(loss_out_dev, tail + LFMQ_TAIL_UQ_LOSS_LAST_TAR, sizeof(float),
                                    cudaMemcpyDeviceToDevice, (cudaStream_t)stream));
    LFMQ_CUDA_CHECK(cudaMemcpyAsync(loss_out_dev + 1, tail + LFMQ_TAIL_MSE0, sizeof(float), cudaMemcpyDeviceToDevice,
                                    (cudaStream_t)stream));
  }
  return LFMQ_OK;
}

// ---- forecast_steps > 1 (rnn_point_estimate.py:109-150) -------------------------------------------------------
namespace {
// Stage 0 is the trunk (num_layers layers + OUTPUT_1); stage s >= 1 one more recurrent layer + BatchNormalization +
// Dropout + OUTPUT_{s+1} on the raw feature width.  All stages share T, F, O and the head: point estimate in every stage,
// or in every stage the uq heads OUTPUT_TARGET_{s+1} / OUTPUT_VARIANCE_{s+1} (rnn_uq_range_estimate.py:114-157).
int chain_check(const lfmq_handle* st, int32_t S, int32_t B, bool training) {
  if (!st || S < 1 || S > lfmq::LFMQ_MAX_STAGES) {
    LFMQ_SET_ERR("lfmq_chain: n_stages %d outside [1, %d]", S, lfmq::LFMQ_MAX_STAGES);
    return LFMQ_ERR_ARG;
  }
  for (int i = 0; i < S; ++i) {
    RUN(check_batch(st[i], B));
    RUN(refuse_dense(st[i], "lfmq_chain"));
    const lfmq_config& c = st[i]->cfg;
    const lfmq_config& c0 = st[0]->cfg;
    if (c.seq_len != c0.seq_len || c.n_inputs != c0.n_inputs || c.n_outputs != c0.n_outputs || c.uq != c0.uq ||
        (i > 0 && c.num_layers != 1)) {
      LFMQ_SET_ERR("lfmq_chain: stage %d does not continue stage 0 (same T/F/O, one layer, same uq flag)", i);
      return LFMQ_ERR_ARG;
    }
    if ((training || c.train) && st[i]->path != Path::Fp32) {
      LFMQ_SET_ERR("lfmq_chain: training-mode stages run on the fp32 or tf32 kernels (stage %d has precision %d)", i,
                   c.precision);
      return LFMQ_ERR_UNSUPPORTED;
    }
    if (training && c.forward_only) {
      LFMQ_SET_ERR("lfmq_chain: stage %d was created forward_only", i);
      return LFMQ_ERR_UNSUPPORTED;
    }
    // the Philox stream index continues after the trunk's layers: the extra layer of stage i is layer L0 + i - 1
    st[i]->tc.stream_base = (i == 0) ? 0 : 2 * (c0.num_layers + i - 1);
  }
  return 0;
}
}  // namespace

int32_t lfmq_chain_forward(const lfmq_handle* stages, int32_t n_stages, const float* x, int32_t B, int64_t row0,
                           int64_t step, float* const* preds, float* work, void* stream) {
  RUN(chain_check(stages, n_stages, B, false));
  if (!x || !preds || (n_stages > 1 && !work)) {
    LFMQ_SET_ERR("lfmq_chain_forward: null pointer");
    return LFMQ_ERR_ARG;
  }
  if (stages[0]->cfg.uq) {
    LFMQ_SET_ERR("lfmq_chain_forward: uq chain, call lfmq_chain_forward_uq");
    return LFMQ_ERR_ARG;
  }
  for (int i = 0; i < n_stages; ++i)
    if (!preds[i]) {
      LFMQ_SET_ERR("lfmq_chain_forward: preds[%d] == NULL", i);
      return LFMQ_ERR_ARG;
    }
  return run_stages(stages, n_stages, x, B, row0, step, preds, nullptr, work, (cudaStream_t)stream);
}

int32_t lfmq_chain_forward_uq(const lfmq_handle* stages, int32_t n_stages, const float* x, int32_t B, int64_t row0,
                              int64_t step, float* const* preds, float* const* vars, float* work, void* stream) {
  RUN(chain_check(stages, n_stages, B, false));
  if (!x || !preds || !vars || (n_stages > 1 && !work)) {
    LFMQ_SET_ERR("lfmq_chain_forward_uq: null pointer");
    return LFMQ_ERR_ARG;
  }
  if (!stages[0]->cfg.uq) {
    LFMQ_SET_ERR("lfmq_chain_forward_uq: point-estimate chain, call lfmq_chain_forward");
    return LFMQ_ERR_ARG;
  }
  for (int i = 0; i < n_stages; ++i)
    if (!preds[i] || !vars[i]) {
      LFMQ_SET_ERR("lfmq_chain_forward_uq: preds[%d] or vars[%d] == NULL", i, i);
      return LFMQ_ERR_ARG;
    }
  return run_stages(stages, n_stages, x, B, row0, step, preds, vars, work, (cudaStream_t)stream);
}

// ---- Monte-Carlo dropout samples of a uq model (lfmq_forward_uq_mc, lfmq_chain_forward_uq_mc) ----------------------
namespace {
// The stages of a forecast analysis, 1 <= S <= LFMQ_MAX_STAGES of them (the caller checks S beside its own sizes):
// non-null handles of one chain, or one dense handle as a model of one stage.  With `chain`, chain_check numbers the
// stages' dropout streams; without it a single handle keeps its own tc.stream_base.  *max_rows: the smallest
// max_batch, the rows one launch may hold.
int stages_check(const lfmq_handle* st, int32_t S, bool chain, const char* fn, int* max_rows) {
  for (int i = 0; i < S; ++i)
    if (!st[i]) {
      LFMQ_SET_ERR("%s: stage %d is a null handle", fn, i);
      return LFMQ_ERR_ARG;
    }
  if (st[0]->path == Path::Dense && S != 1) {
    LFMQ_SET_ERR("%s: a dense handle is a model of one stage (got n_stages %d)", fn, S);
    return LFMQ_ERR_ARG;
  }
  if (chain && st[0]->path != Path::Dense) RUN(chain_check(st, S, 1, false));
  int mb = st[0]->cfg.max_batch;
  for (int i = 1; i < S; ++i) mb = std::min(mb, (int)st[i]->cfg.max_batch);
  *max_rows = mb;
  return 0;
}

// The sizes, uq handles only, then stages_check.  Rows per launch: at most the smallest max_batch.
int mc_check(const lfmq_handle* st, int32_t S, int32_t B, int32_t samples, bool chain, const char* fn,
             int* chunk_max) {
  if (!st || S < 1 || S > lfmq::LFMQ_MAX_STAGES || B < 1 || samples < 1) {
    LFMQ_SET_ERR("%s: need 1 <= n_stages <= %d, B >= 1 and samples >= 1 (got %d, %d, %d)", fn, lfmq::LFMQ_MAX_STAGES, S,
                 B, samples);
    return LFMQ_ERR_ARG;
  }
  for (int i = 0; i < S; ++i)
    if (!st[i] || !st[i]->cfg.uq) {
      LFMQ_SET_ERR("%s: stage %d is not a uq handle: only RNNUqRangeEstimate keeps dropout on at prediction time, a "
                   "point-estimate model would give the same prediction for every sample", fn, i);
      return LFMQ_ERR_ARG;
    }
  return stages_check(st, S, chain, fn, chunk_max);
}

size_t mc_rows(int B, int samples, int chunk_max) {
  return (size_t)std::min<int64_t>((int64_t)samples * B, chunk_max);
}

// Caller scratch for `rows` replicated rows per launch: the replicated input and the chain's next-stage windows
// (win[0], and win[1 ..] read by run_stages as one array), then every stage's sampled preds and vars (m.pred, m.var).
// With dist_elems > 0 (lfmq_chain_forward_uq_dist, B * samples) every stage's gathered samples mu and v follow.
struct McWork {
  float* win[lfmq::LFMQ_MAX_STAGES];
  lfmq::McMoments m;
  lfmq::ChainPtrs mu, v;
};
McWork mc_layout(const lfmq_config& c, int S, size_t rows, size_t dist_elems, Carver& cv) {
  McWork w{};
  for (int i = 0; i < S; ++i) w.win[i] = cv.take<float>(rows * c.seq_len * c.n_inputs);
  for (int i = 0; i < S; ++i) {
    w.m.pred.p[i] = cv.take<float>(rows * c.seq_len * c.n_outputs);
    w.m.var.p[i] = cv.take<float>(rows * c.seq_len * c.n_outputs);
  }
  if (dist_elems)
    for (int i = 0; i < S; ++i) {
      w.mu.p[i] = cv.take<float>(dist_elems);
      w.v.p[i] = cv.take<float>(dist_elems);
    }
  return w;
}

// The distribution pass of lfmq_chain_forward_uq_dist, run by mc_run after its last launch
struct DistArgs {
  const float* levels;
  int n_levels;
  const float* const* y;        // nullable
  float* const* quantiles;
  float* const* scores;
};

// The body of both entry points; `chain` numbers the stages' dropout streams.  Sample s of window b is global row
// row0 + s * B + b of the batch tiled `samples` times, so sample 0 is lfmq_(chain_)forward_uq at (step, row0).  The
// tiled rows run in launches of at most chunk_max rows, in row order, and each launch's samples are folded into the
// moments at once.
// With `dist`, each launch's samples at [T-1, target_idx] are also gathered into the work, and after the last launch
// the distribution pass reads them.
int mc_run(const lfmq_handle* st, int S, bool chain, const float* x, int B, int64_t row0, int64_t step, int samples,
           float* const* mean_pred, float* const* mean_var, float* const* var_pred, float* const* var_var, void* work,
           uint64_t work_bytes, cudaStream_t s, const char* fn, const DistArgs* dist = nullptr) {
  int chunk_max = 0;
  RUN(mc_check(st, S, B, samples, chain, fn, &chunk_max));
  for (int i = 0; i < S; ++i)
    if (!mean_pred || !mean_var || !var_pred || !var_var || !mean_pred[i] || !mean_var[i] || !var_pred[i] ||
        !var_var[i]) {
      LFMQ_SET_ERR("%s: null output of stage %d", fn, i);
      return LFMQ_ERR_ARG;
    }
  if (!x) {
    LFMQ_SET_ERR("%s: x == NULL", fn);
    return LFMQ_ERR_ARG;
  }
  const lfmq_config& c = st[0]->cfg;
  const long row_in = (long)c.seq_len * c.n_inputs, row_out = (long)c.seq_len * c.n_outputs;
  const size_t rows = mc_rows(B, samples, chunk_max);
  McWork w;
  const size_t dist_elems = dist ? (size_t)B * samples : 0;
  RUN(carve_work(work, work_bytes, dist ? fn : "forward_uq_mc",
                 [&](Carver& cv) { return mc_layout(c, S, rows, dist_elems, cv); }, &w));
  lfmq::McMoments& m = w.m;
  for (int i = 0; i < S; ++i) {
    m.mean_pred.p[i] = mean_pred[i];
    m.mean_var.p[i] = mean_var[i];
    m.var_pred.p[i] = var_pred[i];
    m.var_var.p[i] = var_var[i];
  }
  const int64_t total = (int64_t)samples * B;
  for (int64_t r0 = 0; r0 < total; r0 += (int64_t)rows) {
    const int n = (int)std::min<int64_t>((int64_t)rows, total - r0);
    const int64_t b0 = r0 % B;
    const float* in = x + b0 * row_in;            // rows of one sample are a slice of x
    if (b0 + n > B) {
      RUN(mc_replicate(s, B, r0, n, row_in, x, w.win[0]));
      in = w.win[0];
    }
    RUN(run_stages(st, S, in, n, row0 + r0, step, m.pred.p, m.var.p, w.win[1], s));
    RUN(mc_moments(s, S, B, (int)row_out, r0, n, samples, m));
    if (dist)
      RUN(dist_gather(s, S, B, (int)row_out, (long)(c.seq_len - 1) * c.n_outputs + c.target_idx, r0, n, samples, m.pred,
                      m.var, w.mu, w.v));
  }
  if (!dist) return 0;
  lfmq::ChainCPtrs y{};
  lfmq::ChainPtrs q{}, sc{};
  for (int i = 0; i < S; ++i) {
    y.p[i] = dist->y ? dist->y[i] : nullptr;
    q.p[i] = dist->quantiles[i];
    sc.p[i] = dist->y ? dist->scores[i] : nullptr;
  }
  return mixture_dist(s, S, B, samples, dist->levels, dist->n_levels, w.mu, w.v, y, row_out,
                      (long)(c.seq_len - 1) * c.n_outputs + c.target_idx, q, sc);
}
}  // namespace

int32_t lfmq_forward_uq_mc_work_bytes(lfmq_handle h, int32_t B, int32_t samples, uint64_t* bytes) {
  return lfmq_chain_forward_uq_mc_work_bytes(&h, 1, B, samples, bytes);
}

int32_t lfmq_chain_forward_uq_mc_work_bytes(const lfmq_handle* stages, int32_t n_stages, int32_t B, int32_t samples,
                                            uint64_t* bytes) {
  const char* fn = "lfmq_forward_uq_mc_work_bytes";
  int mb = 0;
  RUN(mc_check(stages, n_stages, B, samples, false, fn, &mb));
  const size_t rows = mc_rows(B, samples, mb);
  return report_work_bytes(bytes, fn, [&](Carver& cv) { return mc_layout(stages[0]->cfg, n_stages, rows, 0, cv); });
}

int32_t lfmq_forward_uq_mc(lfmq_handle h, const float* x, int32_t B, int64_t row0, int64_t step, int32_t samples,
                           float* mean_pred, float* mean_var, float* var_pred, float* var_var, void* work,
                           uint64_t work_bytes, void* stream) {
  return mc_run(&h, 1, false, x, B, row0, step, samples, &mean_pred, &mean_var, &var_pred, &var_var, work, work_bytes,
                (cudaStream_t)stream, "lfmq_forward_uq_mc");
}

int32_t lfmq_chain_forward_uq_mc(const lfmq_handle* stages, int32_t n_stages, const float* x, int32_t B, int64_t row0,
                                 int64_t step, int32_t samples, float* const* mean_pred, float* const* mean_var,
                                 float* const* var_pred, float* const* var_var, void* work, uint64_t work_bytes,
                                 void* stream) {
  return mc_run(stages, n_stages, true, x, B, row0, step, samples, mean_pred, mean_var, var_pred, var_var, work,
                work_bytes, (cudaStream_t)stream, "lfmq_chain_forward_uq_mc");
}

namespace {
// The levels: 1 <= n_levels <= LFMQ_DIST_MAX_LEVELS of them, strictly increasing inside (0, 1)
int dist_levels_check(const float* levels, int32_t n_levels, const char* fn) {
  if (n_levels < 1 || n_levels > lfmq::LFMQ_DIST_MAX_LEVELS) {
    LFMQ_SET_ERR("%s: need 1 <= n_levels <= %d (got %d)", fn, lfmq::LFMQ_DIST_MAX_LEVELS, n_levels);
    return LFMQ_ERR_ARG;
  }
  if (!levels) {
    LFMQ_SET_ERR("%s: levels == NULL", fn);
    return LFMQ_ERR_ARG;
  }
  for (int k = 0; k < n_levels; ++k)
    if (!(levels[k] > 0.0 && levels[k] < 1.0) || (k > 0 && !(levels[k] > levels[k - 1]))) {
      LFMQ_SET_ERR("%s: levels must be strictly increasing inside (0, 1) (level %d is %g)", fn, k, levels[k]);
      return LFMQ_ERR_ARG;
    }
  return 0;
}
}  // namespace

int32_t lfmq_chain_forward_uq_dist_work_bytes(const lfmq_handle* stages, int32_t n_stages, int32_t B, int32_t samples,
                                              int32_t n_levels, uint64_t* bytes) {
  const char* fn = "lfmq_chain_forward_uq_dist_work_bytes";
  int mb = 0;
  RUN(mc_check(stages, n_stages, B, samples, false, fn, &mb));
  if (n_levels < 1 || n_levels > lfmq::LFMQ_DIST_MAX_LEVELS) {
    LFMQ_SET_ERR("%s: need 1 <= n_levels <= %d (got %d)", fn, lfmq::LFMQ_DIST_MAX_LEVELS, n_levels);
    return LFMQ_ERR_ARG;
  }
  const size_t rows = mc_rows(B, samples, mb);
  return report_work_bytes(bytes, fn, [&](Carver& cv) {
    return mc_layout(stages[0]->cfg, n_stages, rows, (size_t)B * samples, cv);
  });
}

int32_t lfmq_chain_forward_uq_dist(const lfmq_handle* stages, int32_t n_stages, const float* x, const float* const* y,
                                   int32_t B, int64_t row0, int64_t step, int32_t samples, const float* levels,
                                   int32_t n_levels, float* const* mean_pred, float* const* mean_var,
                                   float* const* var_pred, float* const* var_var, float* const* quantiles,
                                   float* const* scores, void* work, uint64_t work_bytes, void* stream) {
  const char* fn = "lfmq_chain_forward_uq_dist";
  int chunk_max = 0;
  RUN(mc_check(stages, n_stages, B, samples, true, fn, &chunk_max));
  RUN(dist_levels_check(levels, n_levels, fn));
  for (int i = 0; i < n_stages; ++i)
    if (!quantiles || !quantiles[i] || (y && (!y[i] || !scores || !scores[i]))) {
      LFMQ_SET_ERR("%s: null quantiles, target or scores of stage %d", fn, i);
      return LFMQ_ERR_ARG;
    }
  const DistArgs dist{levels, n_levels, y, quantiles, scores};
  return mc_run(stages, n_stages, true, x, B, row0, step, samples, mean_pred, mean_var, var_pred, var_var, work,
                work_bytes, (cudaStream_t)stream, fn, &dist);
}

// ---- integrated gradients of the point forecast (lfmq_integrated_gradients) ----------------------------------------
namespace {
// Built with -DLFMQ_IG_PARAM_GRADS (`make alt`), every interpolant's backward also forms the parameter gradients, into
// the handle's gradient buffer: tools/bench_ig.py measures what skipping them saves.  Not a mode to run in.
#ifdef LFMQ_IG_PARAM_GRADS
constexpr bool kIgInputOnly = false;
#else
constexpr bool kIgInputOnly = true;
#endif

int ig_check(lfmq_handle h, int32_t B, int32_t steps, const char* fn) {
  if (!h) {
    LFMQ_SET_ERR("%s: null handle", fn);
    return LFMQ_ERR_ARG;
  }
  RUN(refuse_dense(h, fn));
  const lfmq_config& c = h->cfg;
  if (c.precision == LFMQ_PREC_BF16 || c.precision == LFMQ_PREC_BF16X3) {
    LFMQ_SET_ERR("%s: the bf16 and bf16x3 paths never form the lowest layer's input gradient; attribute through an "
                 "LFMQ_PREC_FP32 or LFMQ_PREC_TF32 handle holding the same parameters", fn);
    return LFMQ_ERR_UNSUPPORTED;
  }
  if (c.forward_only || c.train || c.uq) {
    LFMQ_SET_ERR("%s: needs a point-estimate handle created with forward_only = 0 and train = 0 (got forward_only %d, "
                 "train %d, uq %d): a forward_only handle keeps no backward buffers, and dropout (train = 1, or any uq "
                 "handle) makes the forecast random", fn, c.forward_only, c.train, c.uq);
    return LFMQ_ERR_ARG;
  }
  if (B < 1 || steps < 1) {
    LFMQ_SET_ERR("%s: need B >= 1 and steps >= 1 (got %d, %d)", fn, B, steps);
    return LFMQ_ERR_ARG;
  }
  return 0;
}

size_t ig_rows(const lfmq_config& c, int B, int steps) {
  return (size_t)std::min<int64_t>((int64_t)steps * B, c.max_batch);
}

// Caller scratch for `rows` rows per launch: the scaled inputs and their input gradients.
struct IgWork { float *xs, *dx; };
IgWork ig_layout(const lfmq_config& c, size_t rows, Carver& cv) {
  IgWork w;
  w.xs = cv.take<float>(rows * c.seq_len * c.n_inputs);
  w.dx = cv.take<float>(rows * c.seq_len * c.n_inputs);
  return w;
}
}  // namespace

int32_t lfmq_integrated_gradients_work_bytes(lfmq_handle h, int32_t B, int32_t steps, uint64_t* bytes) {
  const char* fn = "lfmq_integrated_gradients_work_bytes";
  RUN(ig_check(h, B, steps, fn));
  return report_work_bytes(bytes, fn, [&](Carver& cv) { return ig_layout(h->cfg, ig_rows(h->cfg, B, steps), cv); });
}

int32_t lfmq_integrated_gradients(lfmq_handle h, const float* x, int32_t B, int32_t steps, float* attr, float* f_x,
                                  float* f_base, void* work, uint64_t work_bytes, void* stream) {
  const char* fn = "lfmq_integrated_gradients";
  RUN(ig_check(h, B, steps, fn));
  if (!x || !attr || !f_x || !f_base) {
    LFMQ_SET_ERR("%s: null pointer", fn);
    return LFMQ_ERR_ARG;
  }
  const lfmq_config& c = h->cfg;
  const int T = c.seq_len, O = c.n_outputs, ti = c.target_idx;
  const long row_in = (long)T * c.n_inputs;
  const size_t rows = ig_rows(c, B, steps);
  IgWork w;
  RUN(carve_work(work, work_bytes, fn, [&](Carver& cv) { return ig_layout(c, rows, cv); }, &w));
  cudaStream_t s = (cudaStream_t)stream;
  // f(0): a row's forecast depends on that row alone, so one row of zeros gives every window's baseline
  LFMQ_CUDA_CHECK(cudaMemsetAsync(w.xs, 0, row_in * sizeof(float), s));
  RUN(forward_fp32(h, w.xs, 1, 0, 0, h->preds, nullptr, s));
  RUN(ig_pick(s, B, 1, T, O, ti, h->preds, f_base));
  for (int b0 = 0; b0 < B; b0 += c.max_batch) {       // f(x)
    const int n = std::min(B - b0, c.max_batch);
    RUN(forward_fp32(h, x + b0 * row_in, n, 0, 0, h->preds, nullptr, s));
    RUN(ig_pick(s, n, n, T, O, ti, h->preds, f_x + b0));
  }
  // the interpolants: rows [r0, r0 + n) of the batch tiled `steps` times, their input gradients folded in order
  const int64_t total = (int64_t)steps * B;
  for (int64_t r0 = 0; r0 < total; r0 += (int64_t)rows) {
    const int n = (int)std::min<int64_t>((int64_t)rows, total - r0);
    RUN(ig_scale_inputs(s, B, steps, r0, n, row_in, x, w.xs));
    RUN(forward_fp32(h, w.xs, n, 0, 0, h->preds, nullptr, s));
    RUN(ig_seed(s, n, T, O, ti, h->dpred));
    RUN(backward_fp32(h, w.xs, n, s, w.dx, kIgInputOnly));
    RUN(ig_fold(s, B, steps, r0, n, row_in, w.dx, x, attr));
  }
  return LFMQ_OK;
}

// ---- permutation importance and Shapley attributions (lfmq_chain_permutation_importance, lfmq_chain_shapley) -------
namespace {
// S >= 1 point or uq stages of one chain (chain_check numbers their dropout streams), or one dense handle.  Rows per
// launch: N, at most the smallest max_batch.
int pi_check(const lfmq_handle* st, int32_t S, int32_t N, const char* fn, int* rows) {
  if (!st || S < 1 || S > lfmq::LFMQ_MAX_STAGES || N < 1) {
    LFMQ_SET_ERR("%s: need 1 <= n_stages <= %d and N >= 1 (got %d, %d)", fn, lfmq::LFMQ_MAX_STAGES, S, N);
    return LFMQ_ERR_ARG;
  }
  RUN(stages_check(st, S, true, fn, rows));
  *rows = std::min(N, *rows);
  return 0;
}

int col_group_check(const int32_t* col_group, long row_in, int32_t G, const char* fn) {
  for (long c = 0; c < row_in; ++c)
    if (col_group[c] < 0 || col_group[c] >= G) {
      LFMQ_SET_ERR("%s: col_group[%ld] = %d outside [0, G = %d)", fn, c, col_group[c], G);
      return LFMQ_ERR_ARG;
    }
  return 0;
}

long row_in_of(const lfmq_handle* st) { return (long)st[0]->cfg.seq_len * st[0]->cfg.n_inputs; }
long row_out_of(const lfmq_handle* st) {
  const lfmq_config& c = st[0]->cfg;
  return st[0]->path == Path::Dense ? (long)c.n_outputs : (long)c.seq_len * c.n_outputs;
}

// Where a Shapley launch's outputs are folded (shapley_fold): the K value pointers with their row stride and offset,
// the ordering of the sample being run, and the fp64 sums.
struct ShapleyFold {
  lfmq::ShapleySrc src;
  int K;
  long stride, off;
  int G;
  const int32_t* order;  // o_m of the sample being run
  float* prev;
  double *phi, *f_x, *f_bg;
};

// The forward of one copy of x [N, row_in] in launches of at most `rows` windows, in window order.  Launch [a, a + n)
// builds its rows with the columns whose group ranks >= k in `rank` (device int32, indexed by the device col_group cg)
// taken from window perm_index(N, seed, key, rep, i), or forwards x's own rows when rank == nullptr, and runs every
// stage with dropout keyed by row row_base + i.  Predictions (and variances on a uq chain) go to preds / vars at row a
// when `whole` (copy-sized buffers), else at row 0 (launch-sized ones), where `fold` (nullable) folds each launch's
// outputs as copy k into the Shapley sums.
struct CopyForward {
  const lfmq_handle* st;
  int S;
  const float* x;
  int N, rows;
  long row_in, row_out;
  const int32_t* cg;
  uint64_t seed;
  int64_t step;
  float* xin;       // the launch's gathered rows
  float* slots;     // run_stages' windows of stages 1 .. S-1
  float* const* preds;
  float* const* vars;  // nullptr on a point or dense model
  bool whole;
  cudaStream_t s;

  int run(const int32_t* rank, int k, int key, int rep, int64_t row_base, const ShapleyFold* fold) const {
    float* pp[lfmq::LFMQ_MAX_STAGES];
    float* vp[lfmq::LFMQ_MAX_STAGES];
    for (int a = 0; a < N; a += rows) {
      const int n = std::min(rows, N - a);
      const float* in = x + (long)a * row_in;
      if (rank) {
        RUN(perm_importance_gather(s, x, N, row_in, cg, rank, k, seed, key, rep, a, n, xin));
        in = xin;
      }
      const long off = whole ? (long)a * row_out : 0;
      for (int i = 0; i < S; ++i) {
        pp[i] = preds[i] + off;
        vp[i] = vars ? vars[i] + off : nullptr;
      }
      RUN(run_stages(st, S, in, n, row_base + a, step, pp, vars ? vp : nullptr, slots, s));
      if (fold)
        RUN(shapley_fold(s, fold->src, fold->K, fold->stride, fold->off, a, n, k, fold->G, fold->order, fold->prev,
                         fold->phi, fold->f_x, fold->f_bg));
    }
    return 0;
  }
};

// Caller scratch of permutation importance and Shapley: a launch's gathered rows and the chain's next-stage windows
// (win[0], and win[1 ..] read by run_stages as one array), the device copy of col_group, the analysis's tables, and
// every stage's predictions, then variances on a uq chain.
struct CopyWork {
  float* win[lfmq::LFMQ_MAX_STAGES];
  int32_t *cg, *onehot, *order, *rank;
  float* prev;
  double *phi, *f_x, *f_bg;     // Shapley's fp64 sums
  float* pred[lfmq::LFMQ_MAX_STAGES];
  float* var[lfmq::LFMQ_MAX_STAGES];
};

// Permutation importance: col_group with its groups numbered densely, the one-hot rank rows, and one copy's outputs.
CopyWork pi_layout(const lfmq_handle* st, int S, int rows, int N, Carver& cv) {
  const size_t row_in = row_in_of(st), row_out = row_out_of(st);
  CopyWork w{};
  for (int i = 0; i < S; ++i) w.win[i] = cv.take<float>(rows * row_in);
  w.cg = cv.take<int32_t>(row_in);
  w.onehot = cv.take<int32_t>(2 * row_in);
  for (int i = 0; i < S; ++i) w.pred[i] = cv.take<float>(N * row_out);
  if (st[0]->cfg.uq)
    for (int i = 0; i < S; ++i) w.var[i] = cv.take<float>(N * row_out);
  return w;
}

// Shapley: the perm_index keys of the donor windows and of the group orderings (DESIGN.md section 5f)
constexpr int kShapleyDonorKey = 0x40000000, kShapleyOrderKey = 0x40000001;

// Shapley: one output per stage (two on a uq chain: target and variance), one on a dense handle
int shapley_outputs(const lfmq_handle* st, int S) {
  return st[0]->path == Path::Dense ? 1 : (st[0]->cfg.uq ? 2 * S : S);
}

// Shapley: the samples' group orderings and ranks [samples][G] each, prev [N][K], the fp64 sums of phi [N][K][G], f_x
// and f_bg [N][K], and one launch's outputs.
CopyWork shapley_layout(const lfmq_handle* st, int S, int rows, int N, int G, int samples, Carver& cv) {
  const size_t row_in = row_in_of(st), row_out = row_out_of(st), NK = (size_t)N * shapley_outputs(st, S);
  CopyWork w{};
  for (int i = 0; i < S; ++i) w.win[i] = cv.take<float>(rows * row_in);
  w.cg = cv.take<int32_t>(row_in);
  w.order = cv.take<int32_t>((size_t)samples * G);
  w.rank = cv.take<int32_t>((size_t)samples * G);
  w.prev = cv.take<float>(NK);
  w.phi = cv.take<double>(NK * G);
  w.f_x = cv.take<double>(NK);
  w.f_bg = cv.take<double>(NK);
  for (int i = 0; i < S; ++i) w.pred[i] = cv.take<float>(rows * row_out);
  if (st[0]->cfg.uq)
    for (int i = 0; i < S; ++i) w.var[i] = cv.take<float>(rows * row_out);
  return w;
}

// The explained outputs of a launch (Shapley, ALE): the pointers to every stage's predictions, tar_1, var_1, ..,
// tar_S, var_S on a uq chain (Keras list order), read at row stride row_out_of and at explained_off within a row:
// pred[T-1, target_idx] ([target_idx] on a dense handle).
lfmq::ShapleySrc explained_src(const lfmq_handle* st, int S, float* const* pred, float* const* var) {
  lfmq::ShapleySrc src{};
  for (int i = 0; i < S; ++i) {
    if (st[0]->cfg.uq) {
      src.p[2 * i] = pred[i];
      src.p[2 * i + 1] = var[i];
    } else {
      src.p[i] = pred[i];
    }
  }
  return src;
}
long explained_off(const lfmq_handle* st) {
  const lfmq_config& c = st[0]->cfg;
  return st[0]->path == Path::Dense ? c.target_idx : (long)(c.seq_len - 1) * c.n_outputs + c.target_idx;
}

int shapley_args_check(int32_t N, int32_t G, int32_t samples, const char* fn) {
  if (N < 1 || G < 1 || samples < 1) {
    LFMQ_SET_ERR("%s: need N, G and samples >= 1 (got %d, %d, %d)", fn, N, G, samples);
    return LFMQ_ERR_ARG;
  }
  return 0;
}
}  // namespace

int32_t lfmq_chain_permutation_importance_work_bytes(const lfmq_handle* stages, int32_t n_stages, int32_t N,
                                                     uint64_t* bytes) {
  const char* fn = "lfmq_chain_permutation_importance_work_bytes";
  int rows = 0;
  RUN(pi_check(stages, n_stages, N, fn, &rows));
  return report_work_bytes(bytes, fn, [&](Carver& cv) { return pi_layout(stages, n_stages, rows, N, cv); });
}

int32_t lfmq_chain_permutation_importance(const lfmq_handle* stages, int32_t n_stages, const float* x,
                                          const float* const* y, const float* weights, int32_t N,
                                          const int32_t* col_group, int32_t G, int32_t repeats, uint64_t seed,
                                          int64_t step, float* out_dev, void* work, uint64_t work_bytes, void* stream) {
  const char* fn = "lfmq_chain_permutation_importance";
  int rows = 0;
  RUN(pi_check(stages, n_stages, N, fn, &rows));
  const int S = n_stages;
  const lfmq_config& c = stages[0]->cfg;
  const bool uq = c.uq != 0;
  const long row_in = row_in_of(stages), row_out = row_out_of(stages);
  if (G < 1 || repeats < 1) {
    LFMQ_SET_ERR("%s: need G >= 1 and repeats >= 1 (got %d, %d)", fn, G, repeats);
    return LFMQ_ERR_ARG;
  }
  if (!x || !y || !weights || !col_group || !out_dev) {
    LFMQ_SET_ERR("%s: null pointer", fn);
    return LFMQ_ERR_ARG;
  }
  for (int i = 0; i < S; ++i)
    if (!y[i]) {
      LFMQ_SET_ERR("%s: y[%d] == NULL", fn, i);
      return LFMQ_ERR_ARG;
    }
  RUN(col_group_check(col_group, row_in, G, fn));
  CopyWork w;
  RUN(carve_work(work, work_bytes, fn, [&](Carver& cv) { return pi_layout(stages, S, rows, N, cv); }, &w));
  cudaStream_t s = (cudaStream_t)stream;
  // The gather takes group g's columns from the donor through a rank row that is 1 at g and 0 elsewhere.  G may exceed
  // the columns, so the device col_group numbers the D <= row_in groups present densely (u), and the rank row of
  // group g is the window onehot + D - 1 - u(g) of onehot [2D] = e_{D-1}; a group with no columns reads onehot + D,
  // all zeros, and its copy is x.
  std::vector<int32_t> ids(col_group, col_group + row_in);
  std::sort(ids.begin(), ids.end());
  ids.erase(std::unique(ids.begin(), ids.end()), ids.end());
  const int D = (int)ids.size();
  std::vector<int32_t> dense_cg(row_in), hot(2 * D, 0);
  for (long k = 0; k < row_in; ++k)
    dense_cg[k] = (int32_t)(std::lower_bound(ids.begin(), ids.end(), col_group[k]) - ids.begin());
  hot[D - 1] = 1;
  LFMQ_CUDA_CHECK(cudaMemcpyAsync(w.cg, dense_cg.data(), row_in * sizeof(int32_t), cudaMemcpyHostToDevice, s));
  LFMQ_CUDA_CHECK(cudaMemcpyAsync(w.onehot, hot.data(), 2 * D * sizeof(int32_t), cudaMemcpyHostToDevice, s));
  const int64_t copies = 1 + (int64_t)G * repeats;
  LFMQ_CUDA_CHECK(cudaMemsetAsync(out_dev, 0, copies * 3 * sizeof(float), s));
  const CopyForward cf{stages, S, x, N, rows, row_in, row_out, w.cg, seed, step, w.win[0], w.win[1], w.pred,
                       uq ? w.var : nullptr, true, s};
  // copy 0 is the held-out set as it is; copy 1 + g * repeats + r has group g's columns from window pi_{seed,g,r}(i).
  // Every launch keys its rows by window index (row0 = a), so window i draws the same dropout masks in every copy.
  for (int64_t k = 0; k < copies; ++k) {
    const int g = k == 0 ? -1 : (int)((k - 1) / repeats), r = k == 0 ? -1 : (int)((k - 1) % repeats);
    const int32_t* rank = nullptr;
    if (k > 0) {
      const auto it = std::lower_bound(ids.begin(), ids.end(), g);
      rank = w.onehot + (it != ids.end() && *it == g ? D - 1 - (int)(it - ids.begin()) : D);
    }
    RUN(cf.run(rank, 1, g, r, 0, nullptr));
    float* o = out_dev + 3 * k;
    if (uq && S == 1) {
      RUN(lfmq_loss_uq(stages[0], w.pred[0], w.var[0], y[0], N, o, stream));
    } else if (uq) {
      RUN(lfmq_chain_loss_uq(stages, S, w.pred, w.var, y, weights, N, o, stream));
    } else if (S == 1) {
      RUN(lfmq_loss(stages[0], w.pred[0], y[0], N, o, stream));
    } else {
      RUN(lfmq_chain_loss(stages, S, w.pred, y, weights, N, o, stream));
    }
  }
  return LFMQ_OK;
}

int32_t lfmq_chain_shapley_work_bytes(const lfmq_handle* stages, int32_t n_stages, int32_t N, int32_t G,
                                      int32_t samples, uint64_t* bytes) {
  const char* fn = "lfmq_chain_shapley_work_bytes";
  int rows = 0;
  RUN(pi_check(stages, n_stages, N, fn, &rows));
  RUN(shapley_args_check(N, G, samples, fn));
  return report_work_bytes(bytes, fn,
                           [&](Carver& cv) { return shapley_layout(stages, n_stages, rows, N, G, samples, cv); });
}

int32_t lfmq_chain_shapley(const lfmq_handle* stages, int32_t n_stages, const float* x, int32_t N,
                           const int32_t* col_group, int32_t G, int32_t samples, uint64_t seed, int64_t step,
                           float* phi, float* f_x, float* f_bg, void* work, uint64_t work_bytes, void* stream) {
  const char* fn = "lfmq_chain_shapley";
  int rows = 0;
  RUN(pi_check(stages, n_stages, N, fn, &rows));
  RUN(shapley_args_check(N, G, samples, fn));
  const int S = n_stages, M = samples, K = shapley_outputs(stages, S);
  const bool uq = stages[0]->cfg.uq != 0;
  const long row_in = row_in_of(stages), row_out = row_out_of(stages);
  if (!x || !col_group || !phi || !f_x || !f_bg) {
    LFMQ_SET_ERR("%s: null pointer", fn);
    return LFMQ_ERR_ARG;
  }
  RUN(col_group_check(col_group, row_in, G, fn));
  CopyWork w;
  RUN(carve_work(work, work_bytes, fn, [&](Carver& cv) { return shapley_layout(stages, S, rows, N, G, M, cv); }, &w));
  cudaStream_t s = (cudaStream_t)stream;
  ShapleyFold fold{explained_src(stages, S, w.pred, w.var), K, row_out, explained_off(stages), G, nullptr, w.prev,
                   w.phi, w.f_x, w.f_bg};
  // Sample m belongs to pair p = m / 2.  An even sample orders the groups by o[q] = perm_index(G, seed, 0x40000001,
  // p, q); an odd one reverses its partner's ordering (antithetic) and keeps its donors.
  std::vector<int32_t> ord((size_t)M * G), rk((size_t)M * G);
  for (int m = 0; m < M; ++m)
    for (int q = 0; q < G; ++q) {
      int32_t* o = ord.data() + (size_t)m * G;
      o[q] = (m % 2 == 0) ? (int32_t)lfmq::perm_index(G, seed, kShapleyOrderKey, m / 2, (uint32_t)q)
                          : ord[(size_t)(m - 1) * G + (G - 1 - q)];
      rk[(size_t)m * G + o[q]] = q;
    }
  LFMQ_CUDA_CHECK(cudaMemcpyAsync(w.cg, col_group, row_in * sizeof(int32_t), cudaMemcpyHostToDevice, s));
  LFMQ_CUDA_CHECK(cudaMemcpyAsync(w.order, ord.data(), ord.size() * sizeof(int32_t), cudaMemcpyHostToDevice, s));
  LFMQ_CUDA_CHECK(cudaMemcpyAsync(w.rank, rk.data(), rk.size() * sizeof(int32_t), cudaMemcpyHostToDevice, s));
  LFMQ_CUDA_CHECK(cudaMemsetAsync(w.phi, 0, (size_t)N * K * G * sizeof(double), s));
  LFMQ_CUDA_CHECK(cudaMemsetAsync(w.f_x, 0, (size_t)N * K * sizeof(double), s));
  LFMQ_CUDA_CHECK(cudaMemsetAsync(w.f_bg, 0, (size_t)N * K * sizeof(double), s));
  const CopyForward cf{stages, S, x, N, rows, row_in, row_out, w.cg, seed, step, w.win[0], w.win[1], w.pred,
                       uq ? w.var : nullptr, false, s};
  // Copy (m, k) takes the groups ranked >= k in o_m from window d_p(i) = perm_index(N, seed, 0x40000000, p, i): k = 0
  // is the donor, k = G is x itself, forwarded without a gather.  Every launch of sample m keys window i as row
  // m * N + i, so a uq window shares its dropout masks across the copies of one sample.
  for (int m = 0; m < M; ++m) {
    fold.order = w.order + (size_t)m * G;
    for (int k = 0; k <= G; ++k)
      RUN(cf.run(k < G ? w.rank + (size_t)m * G : nullptr, k, kShapleyDonorKey, m / 2, (int64_t)m * N, &fold));
  }
  RUN(shapley_finish(s, (long)N * K * G, w.phi, M, phi));
  RUN(shapley_finish(s, (long)N * K, w.f_x, M, f_x));
  RUN(shapley_finish(s, (long)N * K, w.f_bg, M, f_bg));
  return LFMQ_OK;
}

// ---- accumulated local effects (lfmq_chain_ale) ---------------------------------------------------------------------
namespace {
// Caller scratch of ALE: a launch's rows and the chain's next-stage windows (as CopyWork), the device cols, the sort's
// keys and windows before and after, its segment offsets, the bin ends [G][K+1], every window's bin [G][N], the local
// effects d [N][J], the fp64 bin means [K][J], one launch's outputs, and the sort's temp storage.
struct AleWork {
  float* win[lfmq::LFMQ_MAX_STAGES];
  int32_t* cols;
  lfmq::AleSort sort;
  float* d;
  double* mean;
  float* pred[lfmq::LFMQ_MAX_STAGES];
  float* var[lfmq::LFMQ_MAX_STAGES];
  void* temp;
};
AleWork ale_layout(const lfmq_handle* st, int S, int rows, int N, int G, int K, size_t temp_bytes, Carver& cv) {
  const size_t row_in = row_in_of(st), row_out = row_out_of(st), J = shapley_outputs(st, S), GN = (size_t)G * N;
  AleWork w{};
  for (int i = 0; i < S; ++i) w.win[i] = cv.take<float>(rows * row_in);
  w.cols = cv.take<int32_t>(G);
  w.sort.key = cv.take<float>(GN);
  w.sort.skey = cv.take<float>(GN);
  w.sort.val = cv.take<int32_t>(GN);
  w.sort.sval = cv.take<int32_t>(GN);
  w.sort.off = cv.take<int32_t>(G + 1);
  w.sort.ends = cv.take<int32_t>((size_t)G * (K + 1));
  w.sort.bin_of = cv.take<int32_t>(GN);
  w.d = cv.take<float>(N * J);
  w.mean = cv.take<double>(K * J);
  for (int i = 0; i < S; ++i) w.pred[i] = cv.take<float>(rows * row_out);
  if (st[0]->cfg.uq)
    for (int i = 0; i < S; ++i) w.var[i] = cv.take<float>(rows * row_out);
  w.temp = cv.take<char>(temp_bytes);
  return w;
}

// pi_check, then N, G, K >= 1 with K <= LFMQ_ALE_MAX_BINS and G * N within the sort's int32 item count; *temp_bytes =
// the sort's temp storage.
int ale_check(const lfmq_handle* st, int32_t S, int32_t N, int32_t G, int32_t K, const char* fn, int* rows,
              size_t* temp_bytes) {
  RUN(pi_check(st, S, N, fn, rows));
  if (G < 1 || K < 1 || K > lfmq::LFMQ_ALE_MAX_BINS || (int64_t)G * N > INT32_MAX) {
    LFMQ_SET_ERR("%s: need N, G >= 1 with G * N < 2^31 and 1 <= K <= %d (got %d, %d, %d)", fn,
                 lfmq::LFMQ_ALE_MAX_BINS, N, G, K);
    return LFMQ_ERR_ARG;
  }
  return lfmq::ale_sort_bytes(N, G, temp_bytes);
}
}  // namespace

int32_t lfmq_chain_ale_work_bytes(const lfmq_handle* stages, int32_t n_stages, int32_t N, int32_t G, int32_t K,
                                  uint64_t* bytes) {
  const char* fn = "lfmq_chain_ale_work_bytes";
  int rows = 0;
  size_t tb = 0;
  RUN(ale_check(stages, n_stages, N, G, K, fn, &rows, &tb));
  return report_work_bytes(bytes, fn, [&](Carver& cv) { return ale_layout(stages, n_stages, rows, N, G, K, tb, cv); });
}

int32_t lfmq_chain_ale(const lfmq_handle* stages, int32_t n_stages, const float* x, int32_t N, const int32_t* cols,
                       int32_t G, int32_t K, int64_t step, int32_t* n_bins, float* edges, int32_t* counts, float* ale,
                       float* local_mean, float* local_sd, void* work, uint64_t work_bytes, void* stream) {
  const char* fn = "lfmq_chain_ale";
  int rows = 0;
  size_t tb = 0;
  RUN(ale_check(stages, n_stages, N, G, K, fn, &rows, &tb));
  const int S = n_stages, J = shapley_outputs(stages, S);
  const long row_in = row_in_of(stages), row_out = row_out_of(stages);
  if (!x || !cols || !n_bins || !edges || !counts || !ale || !local_mean || !local_sd) {
    LFMQ_SET_ERR("%s: null pointer", fn);
    return LFMQ_ERR_ARG;
  }
  for (int g = 0; g < G; ++g)
    if (cols[g] < 0 || cols[g] >= row_in) {
      LFMQ_SET_ERR("%s: cols[%d] = %d outside [0, T * F = %ld)", fn, g, cols[g], row_in);
      return LFMQ_ERR_ARG;
    }
  AleWork w;
  RUN(carve_work(work, work_bytes, fn, [&](Carver& cv) { return ale_layout(stages, S, rows, N, G, K, tb, cv); }, &w));
  cudaStream_t s = (cudaStream_t)stream;
  LFMQ_CUDA_CHECK(cudaMemcpyAsync(w.cols, cols, G * sizeof(int32_t), cudaMemcpyHostToDevice, s));
  RUN(ale_bins(s, x, N, row_in, w.cols, G, K, w.temp, tb, w.sort, n_bins, edges, counts));
  // the bins decide which features have copies to run: a feature with fewer than two distinct values has none
  std::vector<int32_t> kg(G);
  LFMQ_CUDA_CHECK(cudaMemcpyAsync(kg.data(), n_bins, G * sizeof(int32_t), cudaMemcpyDeviceToHost, s));
  LFMQ_CUDA_CHECK(cudaStreamSynchronize(s));
  const lfmq::ShapleySrc src = explained_src(stages, S, w.pred, w.var);
  const long off = explained_off(stages);
  // Feature g's two copies set column cols[g] of window i to the upper and the lower edge of its bin.  Every launch
  // keys its rows by window index (row0 = a), so both copies of window i share its dropout masks at `step`.
  for (int g = 0; g < G; ++g) {
    for (int a = 0; kg[g] > 0 && a < N; a += rows) {
      const int n = std::min(rows, N - a);
      for (int upper = 1; upper >= 0; --upper) {
        RUN(ale_gather(s, x, row_in, cols[g], w.sort.bin_of + (size_t)g * N, edges + (size_t)g * (K + 1), upper, a, n,
                       w.win[0]));
        RUN(run_stages(stages, S, w.win[0], n, a, step, w.pred, stages[0]->cfg.uq ? w.var : nullptr, w.win[1], s));
        RUN(ale_pick(s, src, J, row_out, off, a, n, upper, w.d));
      }
    }
    RUN(ale_fold(s, w.sort, n_bins, g, N, K, J, w.d, w.mean, ale, local_mean, local_sd));
  }
  return LFMQ_OK;
}

// ---- training-window attributions (lfmq_influence_*) ----------------------------------------------------------------
namespace {
// Recurrent handles on the fp32 step (LFMQ_PREC_FP32 / LFMQ_PREC_TF32, any cell, point or uq) and dense handles.
int influence_check(lfmq_handle h, int32_t B, const char* fn) {
  if (!h || B < 1) {
    LFMQ_SET_ERR("%s: need a handle and B >= 1 (got B = %d)", fn, B);
    return LFMQ_ERR_ARG;
  }
  if (h->path != Path::Fp32 && h->path != Path::Dense) {
    LFMQ_SET_ERR("%s: precision %d is not explained directly; explain a LFMQ_PREC_FP32 handle with the same parameters",
                 fn, h->cfg.precision);
    return LFMQ_ERR_ARG;
  }
  return 0;
}

// Caller scratch of the feature passes: a dense launch's predictions [rows][O], a uq launch's variance-head
// pre-activations [rows][T][O].
struct InfluenceWork {
  float *pred, *pre;
};
InfluenceWork influence_layout(lfmq_handle h, Carver& cv) {
  const lfmq_config& c = h->cfg;
  const size_t rows = (size_t)c.max_batch;
  InfluenceWork w{};
  if (h->path == Path::Dense) w.pred = cv.take<float>(rows * c.n_outputs);
  if (c.uq) w.pre = cv.take<float>(rows * c.seq_len * c.n_outputs);
  return w;
}

// u != nullptr: the training features u [J][B][D+1]; else the query features aout [B][D+1] and sout [J][B].  Launches of
// at most max_batch rows, each a forward with every dropout off.
int influence_features(lfmq_handle h, const float* x, const float* y, int B, float* u, float* aout, float* sout,
                       const InfluenceWork& w, cudaStream_t s) {
  const lfmq_config& c = h->cfg;
  const int T = c.seq_len, F = c.n_inputs, O = c.n_outputs, H = c.num_hidden;
  const float* P = h->params;
  for (int r0 = 0; r0 < B; r0 += c.max_batch) {
    const int n = std::min(c.max_batch, B - r0);
    const float* xr = x + (size_t)r0 * T * F;
    if (h->path == Path::Dense) {
      RUN(dense_forward(s, xr, n, T * F, O, P + h->pl.oWo, P + h->pl.obo, w.pred));
      if (u)
        RUN(influence_grad(s, n, 2, 1, T * F, O, c.target_idx, c.target_lambda, 0.f, h->huber, h->huber_delta, xr,
                           w.pred, nullptr, nullptr, y + (size_t)r0 * O, r0, B, u));
      else
        RUN(influence_query(s, n, 1, T * F, O, c.target_idx, 0, xr, nullptr, r0, B, aout, sout));
      continue;
    }
    RUN(forward_fp32(h, xr, n, 0, 0, h->preds, h->var, s, /*dropout_off=*/true));
    const float* a = h->layers[c.num_layers - 1].y;
    if (c.uq) {      // the variance head's pre-activation, by the forward's own product
      RUN(gemm(h, s, n * T, O, H, a, H, 1, P + h->pl.oWv, O, 1, w.pre, O, 0.f, nullptr, 0));
      RUN(add_bias_rows(s, (long)n * T, O, w.pre, P + h->pl.obv));
    }
    if (u)
      RUN(influence_grad(s, n, c.uq ? 1 : 0, T, H, O, c.target_idx, c.target_lambda, c.rnn_lambda, 0, 1.f, a, h->preds,
                         h->var, w.pre, y + (size_t)r0 * T * O, r0, B, u));
    else
      RUN(influence_query(s, n, T, H, O, c.target_idx, c.uq, a, w.pre, r0, B, aout, sout));
  }
  return 0;
}

struct TopkWork {
  float* lscore;
  int32_t* lidx;
  double *part, *usum;
};
TopkWork topk_layout(const lfmq::InfluencePlan& pl, Carver& cv) {
  TopkWork w{};
  w.lscore = cv.take<float>(pl.list_elems);
  w.lidx = cv.take<int32_t>(pl.list_elems);
  w.part = cv.take<double>(pl.part_elems);
  w.usum = cv.take<double>(pl.usum_elems);
  return w;
}

int topk_check(int32_t Nq, int32_t Nt, int32_t D1, int32_t J, int32_t K, const char* fn) {
  if (Nq < 1 || Nt < 1 || D1 < 1 || J < 1 || J > 2 || K < 1 || K > lfmq::LFMQ_INFLUENCE_MAX_K) {
    LFMQ_SET_ERR("%s: need Nq, Nt, D1 >= 1, J in {1, 2} and 1 <= K <= %d (got %d, %d, %d, %d, %d)", fn,
                 lfmq::LFMQ_INFLUENCE_MAX_K, Nq, Nt, D1, J, K);
    return LFMQ_ERR_ARG;
  }
  return 0;
}
}  // namespace

int32_t lfmq_influence_features_work_bytes(lfmq_handle h, uint64_t* bytes) {
  const char* fn = "lfmq_influence_features_work_bytes";
  RUN(influence_check(h, 1, fn));
  return report_work_bytes(bytes, fn, [&](Carver& cv) { return influence_layout(h, cv); });
}

int32_t lfmq_influence_train_features(lfmq_handle h, const float* x, const float* y, int32_t B, float* u, void* work,
                                      uint64_t work_bytes, void* stream) {
  const char* fn = "lfmq_influence_train_features";
  RUN(influence_check(h, B, fn));
  if (!x || !y || !u) {
    LFMQ_SET_ERR("%s: null pointer", fn);
    return LFMQ_ERR_ARG;
  }
  InfluenceWork w;
  RUN(carve_work(work, work_bytes, fn, [&](Carver& cv) { return influence_layout(h, cv); }, &w));
  return influence_features(h, x, y, B, u, nullptr, nullptr, w, (cudaStream_t)stream);
}

int32_t lfmq_influence_query_features(lfmq_handle h, const float* x, int32_t B, float* a, float* s, void* work,
                                      uint64_t work_bytes, void* stream) {
  const char* fn = "lfmq_influence_query_features";
  RUN(influence_check(h, B, fn));
  if (!x || !a || !s) {
    LFMQ_SET_ERR("%s: null pointer", fn);
    return LFMQ_ERR_ARG;
  }
  InfluenceWork w;
  RUN(carve_work(work, work_bytes, fn, [&](Carver& cv) { return influence_layout(h, cv); }, &w));
  return influence_features(h, x, nullptr, B, nullptr, a, s, w, (cudaStream_t)stream);
}

int32_t lfmq_influence_topk_work_bytes(int32_t Nq, int32_t Nt, int32_t D1, int32_t J, int32_t K, uint64_t* bytes) {
  const char* fn = "lfmq_influence_topk_work_bytes";
  RUN(topk_check(Nq, Nt, D1, J, K, fn));
  const lfmq::InfluencePlan pl = lfmq::influence_plan(Nq, Nt, D1, J, K);
  return report_work_bytes(bytes, fn, [&](Carver& cv) { return topk_layout(pl, cv); });
}

int32_t lfmq_influence_topk(const float* a, const float* u, const float* s, int32_t Nq, int32_t Nt, int32_t D1,
                            int32_t J, int32_t K, int32_t* pos_idx, float* pos_score, int32_t* neg_idx,
                            float* neg_score, float* total, void* work, uint64_t work_bytes, void* stream) {
  const char* fn = "lfmq_influence_topk";
  RUN(topk_check(Nq, Nt, D1, J, K, fn));
  if (!a || !u || !s || !pos_idx || !pos_score || !neg_idx || !neg_score || !total) {
    LFMQ_SET_ERR("%s: null pointer", fn);
    return LFMQ_ERR_ARG;
  }
  const lfmq::InfluencePlan pl = lfmq::influence_plan(Nq, Nt, D1, J, K);
  TopkWork w;
  RUN(carve_work(work, work_bytes, fn, [&](Carver& cv) { return topk_layout(pl, cv); }, &w));
  return lfmq::influence_topk((cudaStream_t)stream, pl, a, u, s, Nq, Nt, D1, J, K, w.lscore, w.lidx, w.part, w.usum,
                              pos_idx, pos_score, neg_idx, neg_score, total);
}

// ---- nearest pool rows (lfmq_nearest_topk) ------------------------------------------------------------------------
namespace {
struct NearestWork {
  float* lscore;
  int32_t* lidx;
  float* bn;
};
NearestWork nearest_layout(const lfmq::InfluencePlan& pl, int32_t Nt, Carver& cv) {
  NearestWork w{};
  w.lscore = cv.take<float>(pl.list_elems);
  w.lidx = cv.take<int32_t>(pl.list_elems);
  w.bn = cv.take<float>((size_t)Nt);
  return w;
}

// the pool split of the shortlisting GEMM, which keeps nearest_candidates(K) rows per query
lfmq::InfluencePlan nearest_plan(int32_t Nq, int32_t Nt, int32_t D1, int32_t K) {
  return lfmq::influence_plan(Nq, Nt, D1, 1, lfmq::nearest_candidates(K));
}
}  // namespace

int32_t lfmq_nearest_topk_work_bytes(int32_t Nq, int32_t Nt, int32_t D1, int32_t K, uint64_t* bytes) {
  const char* fn = "lfmq_nearest_topk_work_bytes";
  RUN(topk_check(Nq, Nt, D1, 1, K, fn));
  const lfmq::InfluencePlan pl = nearest_plan(Nq, Nt, D1, K);
  return report_work_bytes(bytes, fn, [&](Carver& cv) { return nearest_layout(pl, Nt, cv); });
}

int32_t lfmq_nearest_topk(const float* a, const float* b, const float* value, int32_t Nq, int32_t Nt, int32_t D1,
                          int32_t K, int32_t* idx, float* d2, float* mean, void* work, uint64_t work_bytes,
                          void* stream) {
  const char* fn = "lfmq_nearest_topk";
  RUN(topk_check(Nq, Nt, D1, 1, K, fn));
  if (!a || !b || !idx || !d2 || (!value) != (!mean)) {
    LFMQ_SET_ERR("%s: null pointer (value and mean go together)", fn);
    return LFMQ_ERR_ARG;
  }
  const lfmq::InfluencePlan pl = nearest_plan(Nq, Nt, D1, K);
  NearestWork w;
  RUN(carve_work(work, work_bytes, fn, [&](Carver& cv) { return nearest_layout(pl, Nt, cv); }, &w));
  const cudaStream_t s = (cudaStream_t)stream;
  RUN(lfmq::nearest_norms(s, b, Nt, D1, w.bn));
  return lfmq::nearest_topk(s, pl, a, b, w.bn, value, Nq, Nt, D1, K, w.lscore, w.lidx, idx, d2, mean);
}

// ---- split-conformal intervals (lfmq_conformal_*) -----------------------------------------------------------------
namespace {
int conformal_shape_check(int32_t S, int32_t N, const char* fn) {
  if (S < 1 || N < 1 || (int64_t)S * N > INT32_MAX) {
    LFMQ_SET_ERR("%s: need S, N >= 1 with S * N < 2^31 (got %d, %d)", fn, S, N);
    return LFMQ_ERR_ARG;
  }
  return 0;
}

int conformal_levels_check(const double* levels, int32_t Q, const char* fn) {
  if (!levels || Q < 1 || Q > lfmq::LFMQ_CONFORMAL_MAX_LEVELS) {
    LFMQ_SET_ERR("%s: need 1 <= Q <= %d host levels (got %d)", fn, lfmq::LFMQ_CONFORMAL_MAX_LEVELS, Q);
    return LFMQ_ERR_ARG;
  }
  for (int k = 0; k < Q; ++k)
    if (!(levels[k] > 0.0 && levels[k] < 1.0) || (k > 0 && !(levels[k] > levels[k - 1]))) {
      LFMQ_SET_ERR("%s: the levels must be strictly increasing inside (0, 1)", fn);
      return LFMQ_ERR_ARG;
    }
  return 0;
}

struct ConformalWork {
  uint64_t *key, *skey;
  char* temp;
};
ConformalWork conformal_layout(int32_t S, int32_t Nc, size_t temp_bytes, Carver& cv) {
  ConformalWork w{};
  w.key = cv.take<uint64_t>((size_t)S * Nc);
  w.skey = cv.take<uint64_t>((size_t)S * Nc);
  w.temp = cv.take<char>(temp_bytes);
  return w;
}
}  // namespace

int32_t lfmq_conformal_scores_work_bytes(int32_t S, int32_t N, uint64_t* bytes) {
  const char* fn = "lfmq_conformal_scores_work_bytes";
  RUN(conformal_shape_check(S, N, fn));
  return report_work_bytes(bytes, fn, [](Carver&) { return 0; });
}

int32_t lfmq_conformal_scores(const float* pred, const float* y, const float* scale, int32_t S, int32_t N, float* r,
                              void* work, uint64_t work_bytes, void* stream) {
  const char* fn = "lfmq_conformal_scores";
  RUN(conformal_shape_check(S, N, fn));
  if (!pred || !y || !r) {
    LFMQ_SET_ERR("%s: null pointer", fn);
    return LFMQ_ERR_ARG;
  }
  (void)work;
  (void)work_bytes;
  return lfmq::conformal_scores((cudaStream_t)stream, (long)S * N, pred, y, scale, r);
}

int32_t lfmq_conformal_calibrate_work_bytes(int32_t S, int32_t Nc, uint64_t* bytes) {
  const char* fn = "lfmq_conformal_calibrate_work_bytes";
  RUN(conformal_shape_check(S, Nc, fn));
  size_t temp = 0;
  RUN(lfmq::conformal_sort_bytes(S, Nc, &temp));
  return report_work_bytes(bytes, fn, [&](Carver& cv) { return conformal_layout(S, Nc, temp, cv); });
}

int32_t lfmq_conformal_calibrate(const float* pred, const float* y, const float* scale, int32_t S, int32_t Nc,
                                 const double* levels, int32_t Q, int32_t* n_valid, float* sorted, float* qhat,
                                 void* work, uint64_t work_bytes, void* stream) {
  const char* fn = "lfmq_conformal_calibrate";
  RUN(conformal_shape_check(S, Nc, fn));
  RUN(conformal_levels_check(levels, Q, fn));
  if (!pred || !y || !n_valid || !sorted || !qhat) {
    LFMQ_SET_ERR("%s: null pointer", fn);
    return LFMQ_ERR_ARG;
  }
  size_t temp = 0;
  RUN(lfmq::conformal_sort_bytes(S, Nc, &temp));
  ConformalWork w;
  RUN(carve_work(work, work_bytes, fn, [&](Carver& cv) { return conformal_layout(S, Nc, temp, cv); }, &w));
  return lfmq::conformal_calibrate((cudaStream_t)stream, S, Nc, pred, y, scale, levels, Q, w.temp, temp, w.key, w.skey,
                                   n_valid, sorted, qhat);
}

int32_t lfmq_conformal_apply_work_bytes(int32_t S, int32_t N, int32_t Nc, int32_t Q, uint64_t* bytes) {
  const char* fn = "lfmq_conformal_apply_work_bytes";
  RUN(conformal_shape_check(S, N, fn));
  RUN(conformal_shape_check(S, Nc, fn));
  if (Q < 1 || Q > lfmq::LFMQ_CONFORMAL_MAX_LEVELS) {
    LFMQ_SET_ERR("%s: need 1 <= Q <= %d (got %d)", fn, lfmq::LFMQ_CONFORMAL_MAX_LEVELS, Q);
    return LFMQ_ERR_ARG;
  }
  return report_work_bytes(bytes, fn, [](Carver&) { return 0; });
}

int32_t lfmq_conformal_apply(const float* pred, const float* y, const float* scale, int32_t S, int32_t N,
                             const float* sorted, const int32_t* n_valid, const float* qhat, int32_t Nc, int32_t Q,
                             float* lower, float* upper, float* pvalue, void* work, uint64_t work_bytes,
                             void* stream) {
  const char* fn = "lfmq_conformal_apply";
  uint64_t need = 0;
  RUN(lfmq_conformal_apply_work_bytes(S, N, Nc, Q, &need));
  if (!pred || !sorted || !n_valid || !qhat || !lower || !upper || !pvalue) {
    LFMQ_SET_ERR("%s: null pointer", fn);
    return LFMQ_ERR_ARG;
  }
  (void)work;
  (void)work_bytes;
  return lfmq::conformal_apply((cudaStream_t)stream, S, N, Nc, Q, pred, y, scale, sorted, n_valid, qhat, lower, upper,
                               pvalue);
}

// ---- lookahead factor backtests (lfmq_factor_eval) ----------------------------------------------------------------
namespace {
int factor_check(int32_t N, int32_t D, int32_t G, int32_t M, int32_t Q, const char* fn) {
  if (N < 1 || D < 1 || G < 1 || G > lfmq::LFMQ_FACTOR_MAX_G || M < 1 || M > lfmq::LFMQ_FACTOR_MAX_M || Q < 2 ||
      Q > lfmq::LFMQ_FACTOR_MAX_Q) {
    LFMQ_SET_ERR("%s: need N, D >= 1, 1 <= G <= %d, 1 <= M <= %d and 2 <= Q <= %d (got N %d, D %d, G %d, M %d, Q %d)",
                 fn, lfmq::LFMQ_FACTOR_MAX_G, lfmq::LFMQ_FACTOR_MAX_M, lfmq::LFMQ_FACTOR_MAX_Q, N, D, G, M, Q);
    return LFMQ_ERR_ARG;
  }
  return 0;
}

lfmq::FactorWork factor_layout(int32_t N, int32_t D, int32_t M, size_t temp_bytes, Carver& cv) {
  const size_t n = (size_t)N;
  lfmq::FactorWork w{};
  w.k0 = cv.take<uint64_t>(n);
  w.k1 = cv.take<uint64_t>(n);
  w.gkey = cv.take<uint64_t>(n);
  w.mkey = cv.take<uint64_t>(M * n);
  w.v0 = cv.take<int32_t>(n);
  w.v1 = cv.take<int32_t>(n);
  w.pos = cv.take<int32_t>(n);
  w.d0 = cv.take<uint32_t>(n);
  w.d1 = cv.take<uint32_t>(n);
  w.base_row = cv.take<int32_t>(n);
  w.seg_off = cv.take<int32_t>((size_t)D + 1);
  w.pred = cv.take<int32_t>(n);
  w.mrow = cv.take<int32_t>(M * n);
  w.grow = cv.take<int32_t>(n);
  w.flag = cv.take<int32_t>(n);
  w.pcg = cv.take<int32_t>(M * (n + 1));
  w.pcm = cv.take<int32_t>(n + 1);
  w.yr = cv.take<uint32_t>(M * n);
  w.bq = cv.take<uint8_t>(n);
  w.temp = cv.take<char>(temp_bytes);
  return w;
}
}  // namespace

int32_t lfmq_factor_eval_work_bytes(int32_t N, int32_t D, int32_t G, int32_t M, int32_t Q, uint64_t* bytes) {
  const char* fn = "lfmq_factor_eval_work_bytes";
  RUN(factor_check(N, D, G, M, Q, fn));
  if (!bytes) {
    LFMQ_SET_ERR("%s: bytes == NULL", fn);
    return LFMQ_ERR_ARG;
  }
  size_t temp = 0;
  RUN(lfmq::factor_temp_bytes(N, D, &temp));
  return report_work_bytes(bytes, fn, [&](Carver& cv) { return factor_layout(N, D, M, temp, cv); });
}

int32_t lfmq_factor_eval(const int32_t* date_idx, const int32_t* company, int32_t N, int32_t D, const double* score,
                         int32_t G, const double* measure, int32_t M, int32_t Q, int32_t* n, int32_t* bucket_n,
                         int32_t* n_pair, double* ic, double* bucket_mean, double* spread, double* turnover, void* work,
                         uint64_t work_bytes, void* stream) {
  const char* fn = "lfmq_factor_eval";
  RUN(factor_check(N, D, G, M, Q, fn));
  if (!date_idx || !company || !score || !measure || !n || !bucket_n || !n_pair || !ic || !bucket_mean || !spread ||
      !turnover) {
    LFMQ_SET_ERR("%s: null pointer", fn);
    return LFMQ_ERR_ARG;
  }
  size_t temp = 0;
  RUN(lfmq::factor_temp_bytes(N, D, &temp));
  lfmq::FactorWork w;
  RUN(carve_work(work, work_bytes, fn, [&](Carver& cv) { return factor_layout(N, D, M, temp, cv); }, &w));
  const lfmq::FactorOut o{n, bucket_n, n_pair, ic, bucket_mean, spread, turnover};
  return lfmq::factor_eval((cudaStream_t)stream, date_idx, company, N, D, score, G, measure, M, Q, w, temp, o);
}

int32_t lfmq_chain_loss(const lfmq_handle* stages, int32_t n_stages, const float* const* preds, const float* const* y,
                        const float* weights, int32_t B, float* out_dev, void* stream) {
  if (!stages || n_stages < 1 || n_stages > lfmq::LFMQ_MAX_STAGES || !preds || !y || !weights || !out_dev || B <= 0) {
    LFMQ_SET_ERR("lfmq_chain_loss: bad argument");
    return LFMQ_ERR_ARG;
  }
  cudaStream_t s = (cudaStream_t)stream;
  lfmq::ChainPtrs none{}, l2{};
  lfmq::ChainWeights w{};
  for (int i = 0; i < n_stages; ++i) {
    if (!stages[i]) {
      LFMQ_SET_ERR("lfmq_chain_loss: null handle");
      return LFMQ_ERR_ARG;
    }
    RUN(refuse_dense(stages[i], "lfmq_chain_loss"));
    l2.p[i] = stages[i]->sc->chain_loss;
    RUN(lfmq_loss(stages[i], preds[i], y[i], B, l2.p[i], stream));
    w.w[i] = weights[i];
  }
  return chain_combine(s, n_stages, none, 0.f, l2, w, out_dev);
}

int32_t lfmq_chain_loss_uq(const lfmq_handle* stages, int32_t n_stages, const float* const* preds,
                           const float* const* vars, const float* const* y, const float* weights, int32_t B,
                           float* out_dev, void* stream) {
  if (!stages || n_stages < 1 || n_stages > lfmq::LFMQ_MAX_STAGES || !preds || !vars || !y || !weights || !out_dev ||
      B <= 0) {
    LFMQ_SET_ERR("lfmq_chain_loss_uq: bad argument");
    return LFMQ_ERR_ARG;
  }
  lfmq::ChainUqArgs a{};
  for (int i = 0; i < n_stages; ++i) {
    if (!stages[i] || !stages[i]->cfg.uq || !preds[i] || !vars[i] || !y[i]) {
      LFMQ_SET_ERR("lfmq_chain_loss_uq: stage %d: null pointer or a point-estimate handle", i);
      return LFMQ_ERR_ARG;
    }
    a.pred.p[i] = const_cast<float*>(preds[i]);
    a.var.p[i] = const_cast<float*>(vars[i]);
    a.y.p[i] = const_cast<float*>(y[i]);
    a.w.w[i] = weights[i];
  }
  const lfmq_config& c = stages[0]->cfg;
  return chain_uq_loss_grad((cudaStream_t)stream, n_stages, B, c.seq_len, c.n_outputs, a, c.target_idx, c.target_lambda,
                            c.rnn_lambda, out_dev, stages[0]->scratch);
}

namespace {
int chain_backward(const lfmq_handle* stages, int32_t n_stages, const float* x, const float* const* y,
                   const float* weights, int32_t B, int64_t row0, int64_t step, const float* denom, float* work,
                   float* loss_out_dev, void* stream) {
  RUN(chain_check(stages, n_stages, B, true));
  if (!x || !y || !weights || !work) {
    LFMQ_SET_ERR("lfmq_chain_backward: null pointer");
    return LFMQ_ERR_ARG;
  }
  for (int i = 0; i < n_stages; ++i)
    if (!y[i]) {
      LFMQ_SET_ERR("lfmq_chain_backward: y[%d] == NULL", i);
      return LFMQ_ERR_ARG;
    }
  return backward_stages(stages, n_stages, x, y, weights, B, row0, step, denom, work, loss_out_dev,
                         (cudaStream_t)stream);
}

// the handles whose gradients one flat vector carries: all trainable, all of one kind (uq or point estimate)
int pack_check(const lfmq_handle* st, int32_t S, const char* fn, lfmq::GradPack* p, int64_t* total) {
  if (!st || S < 1 || S > lfmq::LFMQ_MAX_STAGES) {
    LFMQ_SET_ERR("%s: n_stages %d outside [1, %d]", fn, S, lfmq::LFMQ_MAX_STAGES);
    return LFMQ_ERR_ARG;
  }
  int64_t off = 0;
  for (int i = 0; i < S; ++i) {
    if (!st[i] || st[i]->cfg.forward_only || st[i]->cfg.uq != st[0]->cfg.uq || st[i]->path == Path::Dense) {
      LFMQ_SET_ERR("%s: stage %d is null, forward_only, a dense handle or of another kind than stage 0", fn, i);
      return LFMQ_ERR_ARG;
    }
    p->g[i] = st[i]->grads;
    p->n[i] = st[i]->n_train;
    p->off[i] = off;
    off += st[i]->n_train + (st[0]->cfg.uq ? 3 : 2);
  }
  p->ntail = st[0]->cfg.uq ? 3 : 2;
  *total = off;
  return 0;
}
}  // namespace

int32_t lfmq_chain_backward(const lfmq_handle* stages, int32_t n_stages, const float* x, const float* const* y,
                            const float* weights, int32_t B, int64_t row0, int64_t step, float* work,
                            float* loss_out_dev, void* stream) {
  return chain_backward(stages, n_stages, x, y, weights, B, row0, step, nullptr, work, loss_out_dev, stream);
}

int32_t lfmq_chain_backward_dp(const lfmq_handle* stages, int32_t n_stages, const float* x, const float* const* y,
                               const float* weights, int32_t B, int64_t row0, int64_t step, const float* denom_dev,
                               float* work, float* loss_out_dev, void* stream) {
  if (!denom_dev) {
    LFMQ_SET_ERR("lfmq_chain_backward_dp: denom_dev == NULL (lfmq_chain_backward takes this batch's own counts)");
    return LFMQ_ERR_ARG;
  }
  return chain_backward(stages, n_stages, x, y, weights, B, row0, step, denom_dev, work, loss_out_dev, stream);
}

int32_t lfmq_chain_mask_count(const lfmq_handle* stages, int32_t n_stages, const float* const* y, int32_t B,
                              float* out_dev, void* stream) {
  RUN(chain_check(stages, n_stages, B, false));
  if (!y || !out_dev) {
    LFMQ_SET_ERR("lfmq_chain_mask_count: null pointer");
    return LFMQ_ERR_ARG;
  }
  for (int i = 0; i < n_stages; ++i)
    if (!y[i]) {
      LFMQ_SET_ERR("lfmq_chain_mask_count: y[%d] == NULL", i);
      return LFMQ_ERR_ARG;
    }
  return stage_counts(stages, n_stages, y, B, out_dev, (cudaStream_t)stream);
}

int32_t lfmq_chain_grad_pack_size(const lfmq_handle* stages, int32_t n_stages, int64_t* n_elems) {
  lfmq::GradPack p{};
  int64_t n = 0;
  RUN(pack_check(stages, n_stages, "lfmq_chain_grad_pack_size", &p, &n));
  if (!n_elems) {
    LFMQ_SET_ERR("lfmq_chain_grad_pack_size: n_elems == NULL");
    return LFMQ_ERR_ARG;
  }
  *n_elems = n;
  return LFMQ_OK;
}

int32_t lfmq_chain_grad_pack(const lfmq_handle* stages, int32_t n_stages, float* flat, void* stream) {
  lfmq::GradPack p{};
  int64_t n = 0;
  RUN(pack_check(stages, n_stages, "lfmq_chain_grad_pack", &p, &n));
  if (!flat || (reinterpret_cast<uintptr_t>(flat) & 15) != 0) {
    LFMQ_SET_ERR("lfmq_chain_grad_pack: flat must be a 16-byte aligned device pointer");
    return LFMQ_ERR_ARG;
  }
  return grad_pack((cudaStream_t)stream, n_stages, p, flat, false, lfmq::ChainWeights{}, nullptr);
}

int32_t lfmq_chain_grad_unpack(const lfmq_handle* stages, int32_t n_stages, const float* flat, const float* weights,
                               float* loss_out_dev, void* stream) {
  lfmq::GradPack p{};
  int64_t n = 0;
  RUN(pack_check(stages, n_stages, "lfmq_chain_grad_unpack", &p, &n));
  if (!flat || (reinterpret_cast<uintptr_t>(flat) & 15) != 0 || (loss_out_dev && !weights)) {
    LFMQ_SET_ERR("lfmq_chain_grad_unpack: flat must be a 16-byte aligned device pointer; loss_out_dev needs weights");
    return LFMQ_ERR_ARG;
  }
  lfmq::ChainWeights w{};
  for (int i = 0; i < n_stages && weights; ++i) w.w[i] = weights[i];
  return grad_pack((cudaStream_t)stream, n_stages, p, const_cast<float*>(flat), true, w, loss_out_dev);
}

int32_t lfmq_chain_apply(const lfmq_handle* stages, int32_t n_stages, float lr, int64_t iteration, void* stream) {
  if (!stages || n_stages < 1 || n_stages > lfmq::LFMQ_MAX_STAGES) {
    LFMQ_SET_ERR("lfmq_chain_apply: bad argument");
    return LFMQ_ERR_ARG;
  }
  cudaStream_t s = (cudaStream_t)stream;
  lfmq::ChainPtrs sc{}, none{};
  lfmq::ChainWeights w{};
  for (int i = 0; i < n_stages; ++i) {
    lfmq_handle h = stages[i];
    if (!h || h->cfg.forward_only || h->path == Path::Dense) {
      LFMQ_SET_ERR("lfmq_chain_apply: bad handle (null, forward_only or dense)");
      return LFMQ_ERR_ARG;
    }
    float* tail = h->grads + h->n_train;
    RUN(grad_norm_scale(s, h->n_train, h->grads, 0.f, tail + LFMQ_TAIL_GRAD_NORM, h->scratch, &h->sc->norm_ticket));
    sc.p[i] = tail + LFMQ_TAIL_GRAD_NORM;     // ||g_stage||
  }
  // tf.clip_by_global_norm over all stages' variables (train.py:196)
  RUN(chain_combine(s, n_stages, sc, stages[0]->cfg.max_grad_norm, none, w, nullptr));
  for (int i = 0; i < n_stages; ++i) RUN(apply_update(stages[i], lr, iteration, s));
  return LFMQ_OK;
}

int32_t lfmq_profile_enable(lfmq_handle h, int32_t enable) {
  if (!h) {
    LFMQ_SET_ERR("null handle");
    return LFMQ_ERR_ARG;
  }
  Profiler& p = h->prof;
  if (enable && !p.created) {
    for (int r = 0; r < Profiler::kRegions; ++r)
      for (int i = 0; i < Profiler::kCap; ++i) {
        LFMQ_CUDA_CHECK(cudaEventCreate(&p.a[r][i]));
        LFMQ_CUDA_CHECK(cudaEventCreate(&p.b[r][i]));
      }
    p.created = true;
  }
  for (int r = 0; r < Profiler::kRegions; ++r) p.n[r] = 0;
  p.enabled = enable != 0;
  return LFMQ_OK;
}

int32_t lfmq_profile_read(lfmq_handle h, int32_t region, float* total_ms, int32_t* count) {
  if (!h || region < 0 || region >= Profiler::kRegions || !total_ms || !count) {
    LFMQ_SET_ERR("lfmq_profile_read: bad argument");
    return LFMQ_ERR_ARG;
  }
  Profiler& p = h->prof;
  float sum = 0.f;
  for (int i = 0; i < p.n[region]; ++i) {
    LFMQ_CUDA_CHECK(cudaEventSynchronize(p.b[region][i]));
    float ms = 0.f;
    LFMQ_CUDA_CHECK(cudaEventElapsedTime(&ms, p.a[region][i], p.b[region][i]));
    sum += ms;
  }
  *total_ms = sum;
  *count = p.n[region];
  return LFMQ_OK;
}

int32_t lfmq_window_index(const lfmq_window_index_args* a, void* stream) {
  if (!a || a->struct_size != (int32_t)sizeof(lfmq_window_index_args)) {
    LFMQ_SET_ERR("lfmq_window_index_args: struct_size mismatch");
    return LFMQ_ERR_ARG;
  }
  if (!a->key || !a->active || !a->date || !a->inp_idx || !a->tar_idx || !a->rows || !a->count || !a->work) {
    LFMQ_SET_ERR("lfmq_window_index: null pointer");
    return LFMQ_ERR_ARG;
  }
  if (a->n <= 0 || a->cap <= 0 || a->stride <= 0 || a->forecast_n < 0 || a->min_unrollings <= 0 ||
      a->max_unrollings < a->min_unrollings) {
    LFMQ_SET_ERR("lfmq_window_index: bad dimensions");
    return LFMQ_ERR_ARG;
  }
  WindowIndexArgs w;
  w.n = a->n; w.train = a->train; w.stride = a->stride; w.forecast_n = a->forecast_n;
  w.min_steps = a->stride * (a->min_unrollings - 1) + 1;        // data_processing.py:206-207
  w.max_steps = a->stride * (a->max_unrollings - 1) + 1;
  w.start_date = a->start_date; w.end_date = a->end_date; w.last_train_date = a->last_train_date;
  w.key = a->key; w.active = a->active; w.date = a->date;
  return window_index((cudaStream_t)stream, w, a->cap, a->inp_idx, a->tar_idx, a->rows, a->count, a->work);
}

int32_t lfmq_gather_batch(const lfmq_gather_args* a, void* stream) {
  if (!a || a->struct_size != (int32_t)sizeof(lfmq_gather_args)) {
    LFMQ_SET_ERR("lfmq_gather_args: struct_size mismatch");
    return LFMQ_ERR_ARG;
  }
  if (!a->table || !a->inp_idx || !a->tar_idx || !a->inp_cols || !a->fin_cols || !a->center || !a->scale ||
      !a->scale_flag || !a->aux_flag || !a->x || !a->y || !a->seq_norm) {
    LFMQ_SET_ERR("lfmq_gather_batch: null pointer");
    return LFMQ_ERR_ARG;
  }
  if (a->B < 0 || a->T <= 0 || a->F <= 0 || a->O <= 0 || a->O > a->F || a->stride <= 0 || a->n_cols <= 0) {
    LFMQ_SET_ERR("lfmq_gather_batch: bad dimensions");
    return LFMQ_ERR_ARG;
  }
  GatherArgs g;
  g.n_rows = a->n_rows; g.n_cols = a->n_cols; g.B = a->B; g.T = a->T; g.F = a->F; g.O = a->O; g.stride = a->stride;
  g.seq_norm_col = a->seq_norm_col; g.log_squasher = a->log_squasher; g.aux_masking = a->aux_masking;
  g.table = a->table; g.inp_idx = a->inp_idx; g.tar_idx = a->tar_idx; g.inp_cols = a->inp_cols;
  g.fin_cols = a->fin_cols; g.center = a->center; g.scale = a->scale; g.scale_flag = a->scale_flag;
  g.aux_flag = a->aux_flag; g.x = a->x; g.y = a->y; g.seq_norm = a->seq_norm;
  return gather_batch((cudaStream_t)stream, g);
}

int32_t lfmq_row_weights(const double* table, int64_t n_rows, int32_t n_cols, const int32_t* inp_idx, int32_t B,
                         int32_t weight_col, int32_t date_col, double halflife_years, int32_t ref_month, float* w_out,
                         void* stream) {
  if (!table || !inp_idx || !w_out || B < 0 || n_rows <= 0 || n_cols <= 0 || weight_col >= n_cols ||
      date_col < 0 || date_col >= n_cols || halflife_years < 0.0 || (weight_col < 0 && halflife_years == 0.0)) {
    LFMQ_SET_ERR("lfmq_row_weights: null pointer, bad column, negative half-life or no weight source");
    return LFMQ_ERR_ARG;
  }
  return row_weights((cudaStream_t)stream, table, n_cols, inp_idx, B, weight_col, date_col, halflife_years, ref_month,
                     w_out);
}

int32_t lfmq_unscale(const float* in, float* out, int64_t n_rows, int32_t O, const double* scale, const double* center,
                     int32_t log_squasher, void* stream) {
  if (!in || !out || !scale || !center || n_rows < 0 || O <= 0) {
    LFMQ_SET_ERR("lfmq_unscale: bad argument");
    return LFMQ_ERR_ARG;
  }
  return unscale((cudaStream_t)stream, in, out, (long)n_rows, O, scale, center, log_squasher);
}

}  // extern "C"
