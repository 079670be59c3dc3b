// Host launchers of the linear model over the flattened window (dense.cu).  All return 0 or LFMQ_ERR_CUDA.
#pragma once
#include "common.cuh"

namespace lfmq {

// pred[B,O] = x[B,K] W[K,O] + bias[O]
int dense_forward(cudaStream_t s, const float* x, int B, int K, int O, const float* W, const float* bias, float* pred);
// The MLP branch of Losses._get_loss_point_estimate (losses.py:69-75,100-115) over pred, y [B,O]:
// out2 = {target_lambda * mse_0 + (1 - target_lambda) * mse_all, mse_0}, MSE or (huber != 0) Keras Huber terms.
// denom (nullable, device) = {B_global}: both means divide by it (mse_all by B_global * O).  dpred (nullable) =
// dLoss/dpred.  pred == nullptr: out2 = the counts {B, rows whose targets are not all zero}.  rw (nullable): the
// batch's row weights, which weigh every term and count (the counts become {sum of weights, weighted unmasked rows});
// with rw and pred, denom is required.  scratch: dense_loss_scratch(B) floats.
int dense_loss(cudaStream_t s, const float* pred, const float* y, int B, int O, const float* denom, const float* rw,
               int tidx, float lam, int huber, float delta, float* dpred, float* out2, float* scratch);
size_t dense_loss_scratch(long B);
// g[0 : (K+1)*O] = [x^T dpred ; colsum(dpred)]: the kernel gradient [K,O] then the bias gradient [O], through
// dense_wgrad_scratch(B, K, O) floats of row-block partials summed in a fixed order.
int dense_wgrad(cudaStream_t s, const float* x, const float* dpred, int B, int K, int O, float* part, float* g);
size_t dense_wgrad_scratch(int max_batch, int K, int O);

}  // namespace lfmq
