// C-ABI entry points (include/lfmq.h) and step orchestration.
#include "../../include/lfmq.h"

#include <math.h>
#include <stdlib.h>
#include <string.h>

#include <string>
#include <vector>

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

struct LayerBuf {
  float *h, *c, *y, *gates, *rmask;
  // offsets of this layer's tensors in the flat parameter vector
  int64_t oW, oU, ob, ogamma, obeta, omean, ovar;
  int I;
};

}  // namespace

struct lfmq_handle_s {
  lfmq_config cfg;
  std::vector<ParamSpec> specs;
  int64_t n_train, n_total, n_grad_buf;
  int n_slots;
  int64_t oWo, obo;
  int64_t oWv, obv;          // uq: OUTPUT_VARIANCE_1 (oWo/obo are OUTPUT_TARGET_1 then)
  // workspace carve
  float *params, *grads, *slots, *scalars, *denom;
  unsigned int* tickets;
  std::vector<LayerBuf> layers;
  float *z, *hm, *dz, *dy, *dh_out, *hp, *dh_rec, *dc, *dpred, *preds, *scratch;
  float *var, *apre, *da;   // uq only: variance output, its pre-activation, gradient w.r.t. the pre-activation
  float *zh, *dz2;   // GRU only: recurrent projection of one step, gradient w.r.t. the recurrent projection
  size_t scratch_elems;
  lfmq::TcState tc;
  int64_t last_step = 0;     // step and row0 of the last forward: the fp32 backward regenerates that call's dropout masks
  int64_t last_row0 = 0;
  int stream_base = 0;       // first Philox stream index of this handle's layers (stage s of a forecast chain: 2 (L0+s-1))
  int use_gen;               // 1: the general tensor-core path (rnn_tc.cu) runs this handle's bf16 / bf16x3 work
  lfmq::Profiler prof;
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
  if (c->precision != LFMQ_PREC_FP32 && c->precision != LFMQ_PREC_BF16 && c->precision != LFMQ_PREC_BF16X3) {
    LFMQ_SET_ERR("lfmq_config: unknown precision %d", c->precision);
    return LFMQ_ERR_ARG;
  }
  return LFMQ_OK;
}

// Lays out specs + workspace; with base == nullptr only sizes are computed.
size_t layout(lfmq_handle_s* h, char* base) {
  const lfmq_config& c = h->cfg;
  const int H = c.num_hidden, L = c.num_layers, T = c.seq_len, O = c.n_outputs;
  const size_t B = (size_t)c.max_batch;
  h->specs.clear();
  int64_t off = 0;
  auto add = [&](const std::string& name, int ndim, int64_t s0, int64_t s1, int trainable) {
    ParamSpec p{name, ndim, {s0, s1}, off, trainable};
    off += s0 * (ndim == 2 ? s1 : 1);
    h->specs.push_back(p);
    return p.offset;
  };
  h->layers.assign(L, LayerBuf{});
  for (int l = 0; l < L; ++l) {
    LayerBuf& lb = h->layers[l];
    lb.I = (l == 0) ? c.n_inputs : H;
    const bool gru = c.rnn_cell == LFMQ_CELL_GRU;
    const int NG = gru ? 3 : 4;
    const std::string ls = std::string(gru ? "gru_" : "lstm_") + std::to_string(l + 1);
    const std::string bn = (l == 0) ? "batch_normalization" : "batch_normalization_" + std::to_string(l);
    lb.oW = add(ls + "/kernel", 2, lb.I, NG * H, 1);
    lb.oU = add(ls + "/recurrent_kernel", 2, H, NG * H, 1);
    lb.ob = gru ? add(ls + "/bias", 2, 2, 3 * H, 1) : add(ls + "/bias", 1, 4 * H, 1, 1);
    lb.ogamma = add(bn + "/gamma", 1, H, 1, 1);
    lb.obeta = add(bn + "/beta", 1, H, 1, 1);
  }
  if (c.uq) {
    h->oWo = add("OUTPUT_TARGET_1/kernel", 2, H, O, 1);
    h->obo = add("OUTPUT_TARGET_1/bias", 1, O, 1, 1);
    h->oWv = add("OUTPUT_VARIANCE_1/kernel", 2, H, O, 1);
    h->obv = add("OUTPUT_VARIANCE_1/bias", 1, O, 1, 1);
  } else {
    h->oWo = add("OUTPUT_1/kernel", 2, H, O, 1);
    h->obo = add("OUTPUT_1/bias", 1, O, 1, 1);
    h->oWv = h->obv = -1;
  }
  h->n_train = off;
  for (int l = 0; l < L; ++l) {
    const std::string bn = (l == 0) ? "batch_normalization" : "batch_normalization_" + std::to_string(l);
    h->layers[l].omean = add(bn + "/moving_mean", 1, H, 1, 0);
    h->layers[l].ovar = add(bn + "/moving_variance", 1, H, 1, 0);
  }
  h->n_total = off;
  h->n_grad_buf = (h->n_train + 8 + 3) / 4 * 4;
  h->n_slots = (c.optimizer == LFMQ_OPT_ADADELTA || c.optimizer == LFMQ_OPT_ADAM) ? 2 : 1;

  Carver cv{base, 0};
  h->params = cv.take<float>(h->n_total);
  h->grads = cv.take<float>(h->n_grad_buf);
  h->slots = c.forward_only ? nullptr : cv.take<float>((size_t)h->n_slots * h->n_train);
  h->scalars = cv.take<float>(16);
  h->denom = h->scalars + 8;
  h->tickets = reinterpret_cast<unsigned int*>(h->scalars);   // [0] mask count, [1] mask ticket, [2] norm ticket;
                                                              // zeroed at create, every user resets what it used
  const size_t BT = B * T;
  // The fp32 path's activations.  The tensor-core paths carve their own (tc_layout / gen_layout) and never touch these.
  h->z = h->zh = h->hm = h->preds = h->var = h->apre = nullptr;
  h->dz = h->dz2 = h->dy = h->dh_out = h->hp = h->dh_rec = h->dc = h->dpred = h->da = nullptr;
  if (c.precision == LFMQ_PREC_FP32) {
    for (int l = 0; l < L; ++l) {
      LayerBuf& lb = h->layers[l];
      lb.h = cv.take<float>(BT * H);
      lb.c = cv.take<float>(BT * H);
      lb.y = cv.take<float>(BT * H);
      lb.gates = c.forward_only ? nullptr : cv.take<float>(BT * 4 * H);
      lb.rmask = cv.take<float>(B * H);
    }
    h->z = cv.take<float>(B * 4 * H);
    h->zh = (c.rnn_cell == LFMQ_CELL_GRU) ? cv.take<float>(B * 3 * H) : nullptr;
    h->hm = cv.take<float>(B * H);
    h->preds = cv.take<float>(BT * O);
    h->var = c.uq ? cv.take<float>(BT * O) : nullptr;
    h->apre = (c.uq && !c.forward_only) ? cv.take<float>(BT * O) : nullptr;
    if (!c.forward_only) {
      h->dz = cv.take<float>(BT * 4 * H);
      h->dz2 = (c.rnn_cell == LFMQ_CELL_GRU) ? cv.take<float>(BT * 3 * H) : nullptr;
      h->dy = cv.take<float>(BT * H);
      h->dh_out = cv.take<float>(BT * H);
      h->hp = cv.take<float>(BT * H);
      h->dh_rec = cv.take<float>(B * H);
      h->dc = cv.take<float>(B * H);
      h->dpred = cv.take<float>(BT * O);
      h->da = c.uq ? cv.take<float>(BT * O) : nullptr;
    }
  }
  // scratch serves every precision (lfmq_loss, grad_norm_scale)
  size_t scratch = (size_t)4 << 20;
  if (!c.forward_only) {
    const size_t bn_need = ((BT + 127) / 128) * 2 * H + (size_t)1024 * 2 * H;
    if (bn_need > scratch) scratch = bn_need;
  }
  h->scratch_elems = scratch;
  h->scratch = cv.take<float>(scratch);
  // Tensor-core precisions: the persistent cluster kernels (lstm_tc.cu) take the shape family they are specialised for
  // (LSTM, H = 256, one layer, no recurrent dropout; LFMQ_FORCE_GENERIC=1 sends it to the general path as well), every
  // other supported configuration runs the general stepped path (rnn_tc.cu).
  h->use_gen = 0;
  if (c.precision != LFMQ_PREC_FP32) {
    const char* fg = getenv("LFMQ_FORCE_GENERIC");
    const bool force_gen = fg != nullptr && atoi(fg) != 0;
    const bool fast = c.precision == LFMQ_PREC_BF16 && !force_gen && lfmq::tc_shape_supported(c);
    if (!fast) {
      h->use_gen = 1;
      std::vector<lfmq::GenLayerOff> lo(L);
      for (int l = 0; l < L; ++l) {
        const LayerBuf& lb = h->layers[l];
        lo[l] = lfmq::GenLayerOff{lb.oW, lb.oU, lb.ob, lb.ogamma, lb.obeta, lb.omean, lb.ovar, lb.I};
      }
      char why[160];
      if (lfmq::gen_supported(c, why, sizeof(why)))      // lfmq_create reports unsupported configurations (gen_init)
        lfmq::gen_layout(h->tc, c, lo.data(), h->oWo, h->obo, cv);
    } else {
      const LayerBuf& lb = h->layers[0];
      lfmq::tc_layout(h->tc, c, lfmq::TcParamOff{lb.oW, lb.oU, lb.ob, lb.ogamma, lb.obeta, lb.omean, lb.ovar, h->oWo, h->obo},
                      cv);
    }
  }
  return cv.off;
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

// fp32 SIMT forward of all layers; fills layers[l].{h,c,y,(gates)} and `preds`.
// uq handles also fill `var` [B,T,O] (and keep the variance head's pre-activation when a backward pass can follow).
int forward_fp32(lfmq_handle h, const float* x, int B, int64_t row0, int64_t step, float* preds, float* var,
                 cudaStream_t s) {
  const lfmq_config& c = h->cfg;
  const int H = c.num_hidden, T = c.seq_len, O = c.n_outputs, L = c.num_layers;
  const float* P = h->params;
  h->prof.begin(LFMQ_REGION_FWD, s);
  for (int l = 0; l < L; ++l) {
    LayerBuf& lb = h->layers[l];
    const float* in = (l == 0) ? x : h->layers[l - 1].y;
    const int I = lb.I;
    const float* rmask = nullptr;
    const bool stochastic = c.train || c.uq;       // rnn_uq_range_estimate.py:86,88: training=True is a literal there
    if (stochastic && c.recurrent_dropout > 0.f) {
      RUN(gen_row_mask(s, B, H, dropout_key(c.seed, h->stream_base + 2 * l + 1, step, c.recurrent_dropout), row0,
                       lb.rmask));
      rmask = lb.rmask;
    }
    for (int t = 0; t < T && c.rnn_cell == LFMQ_CELL_GRU; ++t) {
      RUN(sgemm(s, B, 3 * H, I, in + (long)t * I, (long)T * I, 1, P + lb.oW, 3 * H, 1, h->z, 3 * H, 0.f, nullptr, 0));
      if (t > 0) {
        const float* hp = rmask ? h->hm : lb.h + (long)(t - 1) * H;
        const long ld = rmask ? H : (long)T * H;
        RUN(sgemm(s, B, 3 * H, H, hp, ld, 1, P + lb.oU, 3 * H, 1, h->zh, 3 * H, 0.f, nullptr, 0));
      }
      RUN(gru_pointwise_fwd(s, B, T, H, t, h->z, t > 0 ? h->zh : nullptr, P + lb.ob, lb.gates, lb.h, rmask,
                            rmask ? h->hm : nullptr));
    }
    for (int t = 0; t < T && c.rnn_cell == LFMQ_CELL_LSTM; ++t) {
      RUN(sgemm(s, B, 4 * H, I, in + (long)t * I, (long)T * I, 1, P + lb.oW, 4 * H, 1, h->z, 4 * H, 0.f, nullptr, 0));
      if (t > 0) {
        const float* hp = rmask ? h->hm : lb.h + (long)(t - 1) * H;
        const long ld = rmask ? H : (long)T * H;
        RUN(sgemm(s, B, 4 * H, H, hp, ld, 1, P + lb.oU, 4 * H, 1, h->z, 4 * H, 1.f, nullptr, 0));
      }
      RUN(lstm_pointwise_fwd(s, B, T, H, t, h->z, P + lb.ob, lb.gates, lb.c, lb.h, rmask, rmask ? h->hm : nullptr));
    }
    const bool drop = stochastic && c.dropout > 0.f;
    RUN(bn_dropout_fwd(s, B, T, H, lb.h, P + lb.ogamma, P + lb.obeta, P + lb.omean, P + lb.ovar, c.bn_epsilon, drop,
                       dropout_key(c.seed, h->stream_base + 2 * l, step, c.dropout), row0, lb.y));
  }
  h->prof.end(LFMQ_REGION_FWD, s);
  h->prof.begin(LFMQ_REGION_HEAD, s);
  const float* yl = h->layers[L - 1].y;
  RUN(sgemm(s, B * T, O, H, yl, H, 1, P + h->oWo, O, 1, preds, O, 0.f, nullptr, 0));
  RUN(add_bias_rows(s, (long)B * T, O, preds, P + h->obo));
  if (c.uq) {
    float* a = h->apre ? h->apre : var;           // forward-only handles activate in place
    RUN(sgemm(s, B * T, O, H, yl, H, 1, P + h->oWv, O, 1, a, O, 0.f, nullptr, 0));
    RUN(add_bias_rows(s, (long)B * T, O, a, P + h->obv));
    RUN(softplus_floor(s, (long)B * T * O, a, var));
  }
  h->prof.end(LFMQ_REGION_HEAD, s);
  return 0;
}

// dx_out (nullable): dLoss/dx [B,T,F] of the lowest layer (the stages of a forecast chain feed predictions back in)
int backward_fp32(lfmq_handle h, const float* x, int B, cudaStream_t s, float* dx_out = nullptr) {
  const lfmq_config& c = h->cfg;
  const int H = c.num_hidden, T = c.seq_len, O = c.n_outputs, L = c.num_layers;
  const long BT = (long)B * T;
  const float* P = h->params;
  float* G = h->grads;
  const float* yl = h->layers[L - 1].y;
  // head: dWo = y^T dpred, dbo = colsum(dpred), dy = dpred Wo^T
  h->prof.begin(LFMQ_REGION_HEAD, s);
  RUN(sgemm(s, H, O, (int)BT, yl, 1, H, h->dpred, O, 1, G + h->oWo, O, 0.f, h->scratch, h->scratch_elems));
  RUN(colsum(s, BT, O, h->dpred, G + h->obo, h->scratch, h->scratch_elems));
  RUN(sgemm(s, (int)BT, H, O, h->dpred, O, 1, P + h->oWo, 1, O, h->dy, H, 0.f, nullptr, 0));
  if (c.uq) {      // variance head: same three products on da, dy accumulates
    RUN(sgemm(s, H, O, (int)BT, yl, 1, H, h->da, O, 1, G + h->oWv, O, 0.f, h->scratch, h->scratch_elems));
    RUN(colsum(s, BT, O, h->da, G + h->obv, h->scratch, h->scratch_elems));
    RUN(sgemm(s, (int)BT, H, O, h->da, O, 1, P + h->oWv, 1, O, h->dy, H, 1.f, nullptr, 0));
  }
  h->prof.end(LFMQ_REGION_HEAD, s);
  for (int l = L - 1; l >= 0; --l) {
    LayerBuf& lb = h->layers[l];
    const int I = lb.I;
    const float* rmask = ((c.train || c.uq) && c.recurrent_dropout > 0.f) ? lb.rmask : nullptr;
    const bool drop = (c.train || c.uq) && c.dropout > 0.f;
    h->prof.begin(LFMQ_REGION_BWD, s);
    RUN(bn_dropout_bwd(s, B, T, H, h->dy, lb.h, P + lb.ogamma, P + lb.omean, P + lb.ovar, c.bn_epsilon, drop,
                       dropout_key(c.seed, h->stream_base + 2 * l, h->last_step, c.dropout), h->last_row0, h->dh_out,
                       G + lb.ogamma, G + lb.obeta, h->scratch, h->scratch_elems));
    const bool gru = c.rnn_cell == LFMQ_CELL_GRU;
    const int NG = gru ? 3 : 4;
    for (int t = T - 1; t >= 0 && gru; --t) {
      RUN(gru_pointwise_bwd(s, B, T, H, t, lb.gates, lb.h, h->dh_out, (t < T - 1) ? h->dh_rec : nullptr, rmask, h->dc,
                            h->dz, h->dz2));
      if (t > 0)
        RUN(sgemm(s, B, H, 3 * H, h->dz2 + (long)t * 3 * H, (long)T * 3 * H, 1, P + lb.oU, 1, 3 * H, h->dh_rec, H, 0.f,
                  nullptr, 0));
    }
    for (int t = T - 1; t >= 0 && !gru; --t) {
      RUN(lstm_pointwise_bwd(s, B, T, H, t, lb.gates, lb.c, h->dh_out, (t < T - 1) ? h->dh_rec : nullptr, rmask, h->dc,
                             h->dz));
      if (t > 0)
        RUN(sgemm(s, B, H, 4 * H, h->dz + (long)t * 4 * H, (long)T * 4 * H, 1, P + lb.oU, 1, 4 * H, h->dh_rec, H, 0.f,
                  nullptr, 0));
    }
    h->prof.end(LFMQ_REGION_BWD, s);
    h->prof.begin(LFMQ_REGION_WGRAD, s);
    const float* in = (l == 0) ? x : h->layers[l - 1].y;
    // LSTM: one gradient buffer feeds dW, dU and db.  GRU: dz = d(input projection), dz2 = d(recurrent projection),
    // bias rows [2][3H] = colsum of each.
    const float* dzr = gru ? h->dz2 : h->dz;
    const int GH = NG * H;
    RUN(sgemm(s, I, GH, (int)BT, in, 1, I, h->dz, GH, 1, G + lb.oW, GH, 0.f, h->scratch, h->scratch_elems));
    RUN(shift_mask(s, B, T, H, lb.h, rmask, h->hp));
    RUN(sgemm(s, H, GH, (int)BT, h->hp, 1, H, dzr, GH, 1, G + lb.oU, GH, 0.f, h->scratch, h->scratch_elems));
    RUN(colsum(s, BT, GH, h->dz, G + lb.ob, h->scratch, h->scratch_elems));
    if (gru) RUN(colsum(s, BT, GH, h->dz2, G + lb.ob + GH, h->scratch, h->scratch_elems));
    if (l > 0 || dx_out)
      RUN(sgemm(s, (int)BT, I, GH, h->dz, GH, 1, P + lb.oW, 1, GH, l > 0 ? h->dy : dx_out, I, 0.f, nullptr, 0));
    h->prof.end(LFMQ_REGION_WGRAD, s);
  }
  return 0;
}

// optimizer update with the clip scale already in the gradient tail (tail[3]) + the MaxNorm kernel constraint
int apply_update(lfmq_handle h, float lr, int64_t iteration, cudaStream_t s) {
  const lfmq_config& c = h->cfg;
  float* tail = h->grads + h->n_train;
  float lr_eff = lr;
  if (c.optimizer == LFMQ_OPT_ADAM) {
    const double t = (double)(iteration + 1);
    lr_eff = (float)((double)lr * sqrt(1.0 - pow(0.999, t)) / (1.0 - pow(0.9, t)));
  }
  RUN(opt_update(s, c.optimizer, h->n_train, h->params, h->grads, h->slots,
                 h->n_slots > 1 ? h->slots + h->n_train : nullptr, tail + 2, lr_eff, 0.f, 0.f, c.sgd_momentum));
  for (int l = 0; l < c.num_layers; ++l)
    RUN(maxnorm_cols(s, h->layers[l].I, (c.rnn_cell == LFMQ_CELL_GRU ? 3 : 4) * c.num_hidden, h->params + h->layers[l].oW,
                     c.max_norm));
  h->tc.weights_dirty = 1;
  return 0;
}

}  // namespace

// =============================================================================================
extern "C" {

const char* lfmq_last_error(void) { return lfmq::g_err; }
int32_t lfmq_abi_version(void) { return LFMQ_ABI_VERSION; }
int64_t lfmq_launch_count(void) { return lfmq::g_launches; }

int32_t lfmq_workspace_bytes(const lfmq_config* cfg, uint64_t* bytes) {
  RUN(validate(cfg));
  if (!bytes) {
    LFMQ_SET_ERR("bytes == NULL");
    return LFMQ_ERR_ARG;
  }
  lfmq_handle_s tmp;
  tmp.cfg = *cfg;
  *bytes = layout(&tmp, nullptr) + WS_ALIGN;
  lfmq::tc_destroy(tmp.tc);
  lfmq::gen_destroy(tmp.tc);
  return LFMQ_OK;
}

int32_t lfmq_create(const lfmq_config* cfg, void* workspace, uint64_t workspace_bytes, lfmq_handle* out) {
  RUN(validate(cfg));
  if (!workspace || !out) {
    LFMQ_SET_ERR("workspace/out == NULL");
    return LFMQ_ERR_ARG;
  }
  lfmq_handle_s* h = new lfmq_handle_s;
  h->cfg = *cfg;
  char* base = reinterpret_cast<char*>(ws_align_up(reinterpret_cast<size_t>(workspace)));
  const size_t need = layout(h, nullptr) + (base - reinterpret_cast<char*>(workspace));
  if (need > workspace_bytes) {
    LFMQ_SET_ERR("workspace too small: need %zu bytes, got %llu", need, (unsigned long long)workspace_bytes);
    delete h;
    return LFMQ_ERR_WORKSPACE;
  }
  layout(h, base);
  h->tc.prof = &h->prof;
  int rc = 0;
  if (h->use_gen) {
    char why[160];
    if (!lfmq::gen_supported(h->cfg, why, sizeof(why))) {
      LFMQ_SET_ERR("tensor-core precision unsupported for this configuration: %s; use LFMQ_PREC_FP32", why);
      rc = LFMQ_ERR_UNSUPPORTED;
    } else {
      rc = lfmq::gen_init(h->tc, h->cfg);
    }
  } else {
    rc = lfmq::tc_init(h->tc, h->cfg);
  }
  if (rc != 0) {
    delete h;
    return rc;
  }
  // zero parameters / gradients / optimizer slots; BN moving_variance = 1
  cudaError_t e = cudaMemsetAsync(h->params, 0, sizeof(float) * h->n_total, 0);
  if (e == cudaSuccess) e = cudaMemsetAsync(h->grads, 0, sizeof(float) * h->n_grad_buf, 0);
  if (e == cudaSuccess && h->slots) e = cudaMemsetAsync(h->slots, 0, sizeof(float) * h->n_slots * h->n_train, 0);
  if (e == cudaSuccess) e = cudaMemsetAsync(h->scalars, 0, sizeof(float) * 16, 0);
  if (e != cudaSuccess) {
    LFMQ_SET_ERR("lfmq_create: memset failed: %s", cudaGetErrorString(e));
    delete h;
    return LFMQ_ERR_CUDA;
  }
  for (int l = 0; l < cfg->num_layers; ++l) {
    rc = lfmq::fill(0, h->params + h->layers[l].ovar, cfg->num_hidden, 1.0f);
    if (rc) {
      delete h;
      return rc;
    }
  }
  e = cudaStreamSynchronize(0);
  if (e != cudaSuccess) {
    LFMQ_SET_ERR("lfmq_create: %s", cudaGetErrorString(e));
    delete h;
    return LFMQ_ERR_CUDA;
  }
  *out = h;
  return LFMQ_OK;
}

int32_t lfmq_destroy(lfmq_handle h) {
  if (h) {
    lfmq::tc_destroy(h->tc);
    lfmq::gen_destroy(h->tc);
    if (h->prof.created)
      for (int r = 0; r < Profiler::kRegions; ++r)
        for (int i = 0; i < Profiler::kCap; ++i) {
          cudaEventDestroy(h->prof.a[r][i]);
          cudaEventDestroy(h->prof.b[r][i]);
        }
    delete h;
  }
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
  if (h->use_gen) return lfmq::gen_forward(h->tc, h->cfg, h->params, x, B, row0, step, preds, s);
  if (h->cfg.precision == LFMQ_PREC_BF16)
    return lfmq::tc_forward(h->tc, h->cfg, h->params, x, B, row0, step, preds, /*save=*/false, s);
  return forward_fp32(h, x, B, row0, step, preds, nullptr, s);
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
  return loss_grad((cudaStream_t)stream, B, c.seq_len, c.n_outputs, preds, y, nullptr, c.target_idx, c.target_lambda,
                   c.rnn_lambda, nullptr, out_dev, nullptr, h->scratch);
}

int32_t lfmq_loss_uq(lfmq_handle h, const float* preds, const float* var, const float* y, int32_t B, float* out_dev,
                     void* stream) {
  if (!h || B <= 0 || !preds || !var || !y || !out_dev) {
    LFMQ_SET_ERR("lfmq_loss_uq: bad handle, batch %d or null pointer", B);
    return LFMQ_ERR_ARG;
  }
  const lfmq_config& c = h->cfg;
  return uq_loss_grad((cudaStream_t)stream, B, c.seq_len, c.n_outputs, preds, var, nullptr, y, nullptr, c.target_idx,
                      c.target_lambda, c.rnn_lambda, nullptr, nullptr, out_dev, out_dev + 1, out_dev + 2, nullptr,
                      h->scratch);
}

int32_t lfmq_mask_count(lfmq_handle h, const float* y, int32_t B, float* out_dev, void* stream) {
  RUN(check_batch(h, B));
  if (!y || !out_dev) {
    LFMQ_SET_ERR("lfmq_mask_count: null pointer");
    return LFMQ_ERR_ARG;
  }
  return mask_count((cudaStream_t)stream, B, h->cfg.seq_len, h->cfg.n_outputs, y, out_dev, h->tickets);
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
  h->last_step = step;
  h->last_row0 = row0;
  if (c.uq) {
    if (denom_dev) {
      LFMQ_SET_ERR("lfmq_backward: data-parallel denominators are not built for uq handles");
      return LFMQ_ERR_UNSUPPORTED;
    }
    float* t = h->grads + h->n_train;
    RUN(forward_fp32(h, x, B, row0, step, h->preds, h->var, s));
    RUN(uq_loss_grad(s, B, c.seq_len, c.n_outputs, nullptr, nullptr, nullptr, y, nullptr, c.target_idx, c.target_lambda,
                     c.rnn_lambda, nullptr, nullptr, nullptr, nullptr, nullptr, h->denom, h->scratch));
    RUN(uq_loss_grad(s, B, c.seq_len, c.n_outputs, h->preds, h->var, h->apre, y, h->denom, c.target_idx, c.target_lambda,
                     c.rnn_lambda, h->dpred, h->da, t, t + 4, t + 1, nullptr, h->scratch));
    return backward_fp32(h, x, B, s);
  }
  const float* denom = denom_dev;
  if (!denom) {
    RUN(mask_count(s, B, c.seq_len, c.n_outputs, y, h->denom, h->tickets));
    denom = h->denom;
  }
  float* tail = h->grads + h->n_train;
  if (h->use_gen) return lfmq::gen_backward(h->tc, c, h->params, h->grads, x, y, B, row0, step, denom, tail, s);
  if (c.precision == LFMQ_PREC_BF16)
    return lfmq::tc_backward(h->tc, c, h->params, h->grads, x, y, B, row0, step, denom, tail, s);
  RUN(forward_fp32(h, x, B, row0, step, h->preds, nullptr, s));
  RUN(loss_grad(s, B, c.seq_len, c.n_outputs, h->preds, y, denom, c.target_idx, c.target_lambda, c.rnn_lambda,
                h->dpred, tail, nullptr, h->scratch));
  return backward_fp32(h, x, B, s);
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
  RUN(grad_norm_scale(s, h->n_train, h->grads, c.max_grad_norm, tail + 2, h->scratch, h->tickets + 2));
  RUN(apply_update(h, lr, iteration, s));
  h->prof.end(LFMQ_REGION_OPT, s);
  return LFMQ_OK;
}

int32_t lfmq_train_step(lfmq_handle h, const float* x, const float* y, int32_t B, int64_t row0, int64_t step, float lr,
                        float* loss_out_dev, void* stream) {
  RUN(lfmq_backward(h, x, y, B, row0, step, nullptr, stream));
  RUN(lfmq_apply(h, lr, step, stream));
  if (loss_out_dev && !h->cfg.uq)
    LFMQ_CUDA_CHECK(cudaMemcpyAsync(loss_out_dev, h->grads + h->n_train, 2 * sizeof(float), cudaMemcpyDeviceToDevice,
                                    (cudaStream_t)stream));
  if (loss_out_dev && h->cfg.uq) {      // {uq_loss_last_tar, mse_0}
    LFMQ_CUDA_CHECK(cudaMemcpyAsync(loss_out_dev, h->grads + h->n_train + 4, sizeof(float), cudaMemcpyDeviceToDevice,
                                    (cudaStream_t)stream));
    LFMQ_CUDA_CHECK(cudaMemcpyAsync(loss_out_dev + 1, h->grads + h->n_train + 1, sizeof(float), cudaMemcpyDeviceToDevice,
                                    (cudaStream_t)stream));
  }
  return LFMQ_OK;
}

// ---- forecast_steps > 1 (rnn_point_estimate.py:109-150) -------------------------------------------------------
namespace {
// Stage 0 is the trunk (num_layers layers + OUTPUT_1); stage s >= 1 one more recurrent layer + BatchNormalization +
// Dropout + OUTPUT_{s+1} on the raw feature width.  All stages share T, F, O.
int chain_check(const lfmq_handle* st, int32_t S, int32_t B, bool training) {
  if (!st || S < 1 || S > lfmq::LFMQ_MAX_STAGES) {
    LFMQ_SET_ERR("lfmq_chain: n_stages %d outside [1, %d]", S, lfmq::LFMQ_MAX_STAGES);
    return LFMQ_ERR_ARG;
  }
  for (int i = 0; i < S; ++i) {
    RUN(check_batch(st[i], B));
    const lfmq_config& c = st[i]->cfg;
    const lfmq_config& c0 = st[0]->cfg;
    if (c.seq_len != c0.seq_len || c.n_inputs != c0.n_inputs || c.n_outputs != c0.n_outputs || c.uq ||
        (i > 0 && c.num_layers != 1)) {
      LFMQ_SET_ERR("lfmq_chain: stage %d does not continue stage 0 (same T/F/O, one layer, point estimate)", i);
      return LFMQ_ERR_ARG;
    }
    if ((training || c.train) && c.precision != LFMQ_PREC_FP32) {
      LFMQ_SET_ERR("lfmq_chain: training-mode stages run on the fp32 kernels (stage %d has precision %d)", i, c.precision);
      return LFMQ_ERR_UNSUPPORTED;
    }
    if (training && c.forward_only) {
      LFMQ_SET_ERR("lfmq_chain: stage %d was created forward_only", i);
      return LFMQ_ERR_UNSUPPORTED;
    }
    // the Philox stream index continues after the trunk's layers: the extra layer of stage i is layer L0 + i - 1
    st[i]->stream_base = (i == 0) ? 0 : 2 * (c0.num_layers + i - 1);
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
  cudaStream_t s = (cudaStream_t)stream;
  const lfmq_config& c = stages[0]->cfg;
  const size_t slot = (size_t)B * c.seq_len * c.n_inputs;
  const float* in = x;
  for (int i = 0; i < n_stages; ++i) {
    if (!preds[i]) {
      LFMQ_SET_ERR("lfmq_chain_forward: preds[%d] == NULL", i);
      return LFMQ_ERR_ARG;
    }
    if (i > 0) {
      float* next = work + (size_t)(i - 1) * slot;
      RUN(chain_next_input(s, B, c.seq_len, c.n_inputs, c.n_outputs, in, preds[i - 1], x, next));
      in = next;
    }
    RUN(lfmq_forward(stages[i], in, B, row0, step, preds[i], stream));
  }
  return LFMQ_OK;
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
    l2.p[i] = stages[i]->scalars + 10;      // two spare floats of the handle's scalar block
    RUN(lfmq_loss(stages[i], preds[i], y[i], B, l2.p[i], stream));
    w.w[i] = weights[i];
  }
  return chain_combine(s, n_stages, none, 0.f, l2, w, out_dev);
}

int32_t lfmq_chain_backward(const lfmq_handle* stages, int32_t n_stages, const float* x, const float* const* y,
                            const float* weights, int32_t B, int64_t row0, int64_t step, float* work,
                            float* loss_out_dev, void* stream) {
  RUN(chain_check(stages, n_stages, B, true));
  if (!x || !y || !weights || !work) {
    LFMQ_SET_ERR("lfmq_chain_backward: null pointer");
    return LFMQ_ERR_ARG;
  }
  cudaStream_t s = (cudaStream_t)stream;
  const int S = n_stages;
  const lfmq_config& c0 = stages[0]->cfg;
  const int T = c0.seq_len, F = c0.n_inputs, O = c0.n_outputs;
  const size_t slot = (size_t)B * T * F;
  float* dx = work + (size_t)(S - 1) * slot;
  // forward of every stage (each keeps its own saved state), then each stage's loss and dLoss/dpred_s, weighted
  lfmq::ChainPtrs dpred{}, l2{}, none{};
  lfmq::ChainWeights w{};
  const float* in = x;
  for (int i = 0; i < S; ++i) {
    lfmq_handle h = stages[i];
    const lfmq_config& c = h->cfg;
    if (!y[i]) {
      LFMQ_SET_ERR("lfmq_chain_backward: y[%d] == NULL", i);
      return LFMQ_ERR_ARG;
    }
    h->last_step = step;
    h->last_row0 = row0;
    if (i > 0) {
      float* next = work + (size_t)(i - 1) * slot;
      RUN(chain_next_input(s, B, T, F, O, in, stages[i - 1]->preds, x, next));
      in = next;
    }
    RUN(forward_fp32(h, in, B, row0, step, h->preds, nullptr, s));
    RUN(mask_count(s, B, T, O, y[i], h->denom, h->tickets));
    float* tail = h->grads + h->n_train;
    RUN(loss_grad(s, B, T, O, h->preds, y[i], h->denom, c.target_idx, c.target_lambda, c.rnn_lambda, h->dpred, tail,
                  nullptr, h->scratch));
    if (weights[i] != 1.0f) RUN(scale_inplace(s, (long)B * T * O, h->dpred, weights[i]));
    dpred.p[i] = h->dpred;
    l2.p[i] = tail;
    w.w[i] = weights[i];
  }
  if (loss_out_dev) RUN(chain_combine(s, S, none, 0.f, l2, w, loss_out_dev));
  // BPTT from the last stage down; the input gradient of stage i lands on the last time step of earlier predictions
  for (int i = S - 1; i >= 1; --i) {
    const float* in_i = work + (size_t)(i - 1) * slot;
    RUN(backward_fp32(stages[i], in_i, B, s, dx));
    RUN(chain_scatter_dx(s, B, T, F, O, i, dx, dpred));
  }
  return backward_fp32(stages[0], x, B, s);
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
    if (!h || h->cfg.forward_only) {
      LFMQ_SET_ERR("lfmq_chain_apply: bad handle");
      return LFMQ_ERR_ARG;
    }
    float* tail = h->grads + h->n_train;
    RUN(grad_norm_scale(s, h->n_train, h->grads, 0.f, tail + 2, h->scratch, h->tickets + 2));   // tail[2] = ||g_stage||
    sc.p[i] = tail + 2;
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

int32_t lfmq_unscale(const float* in, float* out, int64_t n_rows, int32_t O, const double* scale, const double* center,
                     int32_t log_squasher, void* stream) {
  if (!in || !out || !scale || !center || n_rows < 0 || O <= 0) {
    LFMQ_SET_ERR("lfmq_unscale: bad argument");
    return LFMQ_ERR_ARG;
  }
  return unscale((cudaStream_t)stream, in, out, (long)n_rows, O, scale, center, log_squasher);
}

}  // extern "C"
