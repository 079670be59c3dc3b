// bf16 tensor-core path (LFMQ_PREC_BF16): persistent wgmma LSTM forward and backward recurrences, wgmma
// weight-gradient GEMM and the fused HBM-bound head.  See lstm_tc.cu / DESIGN.md.
#pragma once
#include "tc_shared.h"

namespace lfmq {

// The shape family of the persistent cluster kernels: LSTM, point estimate, H = 256, L = 1, F <= 32, O <= 16, no
// recurrent dropout.  Otherwise false, with the reason in why[0 : n].
bool tc_supported(const lfmq_config& cfg, char* why, size_t n);
// Carves the cluster path's buffers from the workspace (only sizes them when the carver has no base).
void tc_layout(TcState& st, const lfmq_config& cfg, Carver& cv);
int tc_init(TcState& st, const lfmq_config& cfg);
void tc_destroy(TcState& st);
// preds may be null (training: the head is fused with the loss in tc_backward)
int tc_forward(TcState& st, const lfmq_config& cfg, const ParamLayout& pl, const float* params, const float* x, int B,
               int64_t row0, int64_t step, float* preds, bool save, cudaStream_t s);
int tc_backward(TcState& st, const lfmq_config& cfg, const ParamLayout& pl, const float* params, float* grads,
                const float* x, const float* y, int B, int64_t row0, int64_t step, const float* denom, float* tail,
                cudaStream_t s);

}  // namespace lfmq
