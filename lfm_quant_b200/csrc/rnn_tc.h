// General tensor-core path (LFMQ_PREC_BF16 for every LSTM point-estimate shape the H=256 / L=1 cluster kernels of
// lstm_tc.cu do not cover, and LFMQ_PREC_BF16X3 everywhere): H in {64, 128, ..., 1024} (multiple of 64), any number of
// stacked layers, dropout and recurrent dropout.  See rnn_tc.cu / DESIGN.md section 5b.
#pragma once
#include "tc_shared.h"

namespace lfmq {

// offsets of one layer's tensors in the flat fp32 parameter / gradient vectors (from layout() in lfmq_api.cu)
struct GenLayerOff {
  int64_t oW, oU, ob, ogamma, obeta, omean, ovar;
  int I;
};

bool gen_supported(const lfmq_config& cfg, char* why, size_t n);
// Carves the general path's buffers from the workspace (only sizes them when the carver has no base).
void gen_layout(TcState& st, const lfmq_config& cfg, const GenLayerOff* layers, int64_t oWo, int64_t obo, Carver& cv);
int gen_init(TcState& st, const lfmq_config& cfg);
void gen_destroy(TcState& st);
// preds [B,T,O] fp32 (predict / validation forward)
int gen_forward(TcState& st, const lfmq_config& cfg, const float* params, const float* x, int B, int64_t row0,
                int64_t step, float* preds, cudaStream_t s);
// forward + loss + BPTT: fills grads[0 : n_trainable] and tail = {loss, mse_0}
int gen_backward(TcState& st, const lfmq_config& cfg, const float* params, float* grads, const float* x,
                 const float* y, int B, int64_t row0, int64_t step, const float* denom, float* tail, cudaStream_t s);

}  // namespace lfmq
