// The linear model over the flattened input window (MLPLinearPointEstimate, mlp_linear_point_estimate.py:66-77):
// pred[B,O] = x[B,K] W[K,O] + b with K = T*F, its MLP-branch loss (losses.py:69-75,100-115) and its gradients.
// fp32 throughout: every kernel streams x once and does O multiply-adds per element, far below the FMA rate, so the
// model is bound by the bytes of x.  Every reduction runs in a fixed order and without atomics: the same inputs give
// the same bits, and a row's prediction depends on that row alone, not on its place in the batch or the batch size.
#include "dense.h"

namespace lfmq {

namespace {

constexpr int kCols = 16;                 // output columns per pass (O > 16 takes several passes)
constexpr int kFwdWarps = 16;            // one CTA per SM, walking the row groups
constexpr int kFwdRowsPerWarp = 4;        // each W element read from shared memory serves four rows
constexpr int kFwdRows = kFwdWarps * kFwdRowsPerWarp;
constexpr int kFwdKChunk = 2048;          // rows of W staged in shared memory at a time (a multiple of 32)
constexpr int kWStride = 20;              // padded row of staged W: the float4 reads of 8 lanes hit distinct banks
constexpr int kLossThreads = 256;
constexpr int kWgThreads = 128;           // k values per weight-gradient block

// pred = x W + b.  A warp owns four rows; lane l accumulates k = l, l + 32, ... in increasing k, then the 32 lane
// sums are combined by one xor butterfly -- the same sequence of operations for every row.  When W fits (T*F <=
// kFwdKChunk, O <= 16) it is staged once and stays in shared memory while the CTA walks its row groups; otherwise each
// (column pass, K chunk) is staged in turn.  The chunk is a multiple of 32, so lane l sums the same k in the same
// order either way.
__global__ void __launch_bounds__(kFwdWarps * 32, 1) dense_fwd_kernel(const float* __restrict__ x, int B, int K, int O,
                                                                     const float* __restrict__ W,
                                                                     const float* __restrict__ bias,
                                                                     float* __restrict__ pred) {
  extern __shared__ __align__(16) float ws[];     // [kFwdKChunk][kWStride]
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const bool resident = K <= kFwdKChunk && O <= kCols;
  const long groups = (B + kFwdRows - 1) / kFwdRows;
  bool staged = false;
  for (long g = blockIdx.x; g < groups; g += gridDim.x) {
    const long row0 = g * kFwdRows + warp * kFwdRowsPerWarp;
    const float* xr[kFwdRowsPerWarp];
    bool live[kFwdRowsPerWarp];
#pragma unroll
    for (int r = 0; r < kFwdRowsPerWarp; ++r) {
      live[r] = row0 + r < B;
      xr[r] = x + (live[r] ? row0 + r : 0) * (long)K;
    }
    for (int c0 = 0; c0 < O; c0 += kCols) {
      const int nc = min(kCols, O - c0);
      float acc[kFwdRowsPerWarp][kCols];
#pragma unroll
      for (int r = 0; r < kFwdRowsPerWarp; ++r)
#pragma unroll
        for (int j = 0; j < kCols; ++j) acc[r][j] = 0.f;
      for (int k0 = 0; k0 < K; k0 += kFwdKChunk) {
        const int nk = min(kFwdKChunk, K - k0);
        if (!(resident && staged)) {
          __syncthreads();
          for (int i = threadIdx.x; i < nk * kCols; i += blockDim.x) {
            const int kk = i / kCols, j = i % kCols;
            ws[kk * kWStride + j] = j < nc ? W[(long)(k0 + kk) * O + c0 + j] : 0.f;
          }
          __syncthreads();
          staged = true;
        }
#pragma unroll 4
        for (int kk = lane; kk < nk; kk += 32) {
          float xv[kFwdRowsPerWarp];
#pragma unroll
          for (int r = 0; r < kFwdRowsPerWarp; ++r) xv[r] = live[r] ? __ldg(xr[r] + k0 + kk) : 0.f;
          const float4* w4 = reinterpret_cast<const float4*>(ws + kk * kWStride);
          float w[kCols];
#pragma unroll
          for (int q = 0; q < kCols / 4; ++q) {
            const float4 v = w4[q];
            w[4 * q] = v.x; w[4 * q + 1] = v.y; w[4 * q + 2] = v.z; w[4 * q + 3] = v.w;
          }
#pragma unroll
          for (int r = 0; r < kFwdRowsPerWarp; ++r)
#pragma unroll
            for (int j = 0; j < kCols; ++j) acc[r][j] = fmaf(xv[r], w[j], acc[r][j]);
        }
      }
#pragma unroll
      for (int r = 0; r < kFwdRowsPerWarp; ++r) {
        float mine = 0.f;
#pragma unroll
        for (int j = 0; j < kCols; ++j) {
          const float v = warp_sum(acc[r][j]);
          if (lane == j) mine = v;
        }
        if (live[r] && lane < nc) pred[(row0 + r) * O + c0 + lane] = mine + bias[c0 + lane];
      }
    }
  }
}

__device__ __forceinline__ float block_sum(float v, float* red) {
  v = warp_sum(v);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  __syncthreads();
  if (lane == 0) red[warp] = v;
  __syncthreads();
  float s = 0.f;
  for (int w = 0; w < (int)(blockDim.x >> 5); ++w) s += red[w];     // every thread, the same order
  return s;
}

// One row per thread.  pred != nullptr: the row's loss terms {f(r_target), sum_o f(r_o)} and, with dpred, the row's
// dLoss/dpred; pred == nullptr: the counts {1, mask}.  With row weights rw (nullable) both are multiplied by the row's
// weight, which scales the first factor of each product (rw = 1 changes no rounding).  Writes the block's two sums to
// part[2 * blockIdx.x].
__global__ void __launch_bounds__(kLossThreads) dense_loss_rows(const float* __restrict__ pred,
                                                                  const float* __restrict__ y, int B, int O,
                                                                  const float* __restrict__ denom,
                                                                  const float* __restrict__ rw, int tidx, float lam,
                                                                  int huber, float delta, float* __restrict__ dpred,
                                                                  float* __restrict__ part) {
  __shared__ float red[kLossThreads / 32];
  const long b = (long)blockIdx.x * blockDim.x + threadIdx.x;
  float s0 = 0.f, sall = 0.f;
  if (b < B) {
    const float* yr = y + b * O;
    const float mask = row_mask(yr, O) ? 1.f : 0.f;          // losses.py:69: ~all(y_true == 0)
    const float wb = row_weight(rw, b);
    if (!pred) {
      s0 = wb;
      sall = mask * wb;
    } else {
      const float bg = denom ? loss_denom(rw, denom[0]) : (float)B;
      const float g_all = (1.f - lam) / (bg * (float)O), g_tar = lam / bg;
      for (int o = 0; o < O; ++o) {
        const float r = yr[o] - pred[b * O + o] * mask;     // losses.py:75: predictions of masked rows are zeroed
        const float ar = fabsf(r);
        float f, df;                                         // f(r) and df/dr
        if (huber && ar > delta) {                           // keras Huber: delta * (|r| - delta / 2)
          f = (delta * wb) * (ar - 0.5f * delta);
          df = copysignf(delta, r);
        } else if (huber) {
          f = (0.5f * wb) * r * r;
          df = r;
        } else {
          f = (r * wb) * r;
          df = 2.f * r;
        }
        sall += f;
        float g = g_all;
        if (o == tidx) {
          s0 = f;
          g += g_tar;
        }
        if (dpred) dpred[b * O + o] = -mask * g * df * wb;
      }
    }
  }
  s0 = block_sum(s0, red);
  sall = block_sum(sall, red);
  if (threadIdx.x == 0) {
    part[2 * blockIdx.x] = s0;
    part[2 * blockIdx.x + 1] = sall;
  }
}

// Sums the n block partials in a fixed order: out = {loss, mse_0} (or the counts {B, mask}).
__global__ void __launch_bounds__(kLossThreads) dense_loss_reduce(const float* __restrict__ part, int n, int B, int O,
                                                                    const float* __restrict__ denom,
                                                                    const float* __restrict__ rw, float lam,
                                                                    int counts, float* __restrict__ out) {
  __shared__ float red[kLossThreads / 32];
  float s0 = 0.f, sall = 0.f;
  for (int i = threadIdx.x; i < n; i += blockDim.x) {
    s0 += part[2 * i];
    sall += part[2 * i + 1];
  }
  s0 = block_sum(s0, red);
  sall = block_sum(sall, red);
  if (threadIdx.x != 0) return;
  if (counts) {
    out[0] = s0;
    out[1] = sall;
    return;
  }
  const float bg = denom ? loss_denom(rw, denom[0]) : (float)B;
  const float mse0 = s0 / bg, mall = sall / (bg * (float)O);   // masked rows count in both denominators
  out[0] = lam * mse0 + (1.f - lam) * mall;
  out[1] = mse0;
}

// Split-K over rows: block (kt, p) sums rows [p * kWgRowsPer, ...) of x[:, k]^T dpred for its kWgThreads values of k.
// k == K is the bias: its x is 1, so the same pass writes db as the last row of the [K + 1][O] partial.
constexpr int kWgRowsPer = 128;
__global__ void __launch_bounds__(kWgThreads) dense_wgrad_partial(const float* __restrict__ x,
                                                                    const float* __restrict__ dpred, int B, int K, int O,
                                                                    float* __restrict__ part) {
  __shared__ float dp[kWgRowsPer * kCols];
  const int k = blockIdx.x * kWgThreads + threadIdx.x;
  const long r0 = (long)blockIdx.y * kWgRowsPer;
  const int nr = (int)min((long)kWgRowsPer, (long)B - r0);
  for (int c0 = 0; c0 < O; c0 += kCols) {
    const int nc = min(kCols, O - c0);
    __syncthreads();
    for (int i = threadIdx.x; i < kWgRowsPer * kCols; i += blockDim.x) {
      const int r = i / kCols, j = i % kCols;
      dp[i] = (r < nr && j < nc) ? dpred[(r0 + r) * O + c0 + j] : 0.f;
    }
    __syncthreads();
    if (k > K) continue;
    float acc[kCols];
#pragma unroll
    for (int j = 0; j < kCols; ++j) acc[j] = 0.f;
    const float* xc = x + r0 * K + k;
#pragma unroll 8
    for (int r = 0; r < nr; ++r) {
      const float xv = k < K ? __ldg(xc + (long)r * K) : 1.f;
#pragma unroll
      for (int j = 0; j < kCols; ++j) acc[j] = fmaf(xv, dp[r * kCols + j], acc[j]);
    }
    float* o = part + ((long)blockIdx.y * (K + 1) + k) * O + c0;
#pragma unroll
    for (int j = 0; j < kCols; ++j)
      if (j < nc) o[j] = acc[j];
  }
}

// g[i] = sum over the n partials, in partial order, of part[p][i]: the [K, O] kernel gradient then the [O] bias one.
__global__ void dense_wgrad_reduce(const float* __restrict__ part, int n, long len, float* __restrict__ g) {
  const long i = (long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= len) return;
  float s = 0.f;
  for (int p = 0; p < n; ++p) s += part[(long)p * len + i];
  g[i] = s;
}

}  // namespace

int dense_forward(cudaStream_t s, const float* x, int B, int K, int O, const float* W, const float* bias, float* pred) {
  constexpr size_t smem = sizeof(float) * kFwdKChunk * kWStride;
  // set on every call: the attribute belongs to the current device, and handles may live on several
  LFMQ_CUDA_CHECK(cudaFuncSetAttribute(dense_fwd_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  const int groups = (B + kFwdRows - 1) / kFwdRows;
  dense_fwd_kernel<<<min(groups, device_sm_count()), kFwdWarps * 32, smem, s>>>(x, B, K, O, W, bias, pred);
  LFMQ_LAUNCH_CHECK();
  return 0;
}

size_t dense_loss_scratch(long B) { return 2 * (size_t)((B + kLossThreads - 1) / kLossThreads); }

int dense_loss(cudaStream_t s, const float* pred, const float* y, int B, int O, const float* denom, const float* rw,
               int tidx, float lam, int huber, float delta, float* dpred, float* out2, float* scratch) {
  const int nb = (B + kLossThreads - 1) / kLossThreads;
  dense_loss_rows<<<nb, kLossThreads, 0, s>>>(pred, y, B, O, denom, rw, tidx, lam, huber, delta, dpred, scratch);
  LFMQ_LAUNCH_CHECK();
  dense_loss_reduce<<<1, kLossThreads, 0, s>>>(scratch, nb, B, O, denom, rw, lam, pred ? 0 : 1, out2);
  LFMQ_LAUNCH_CHECK();
  return 0;
}

size_t dense_wgrad_scratch(int max_batch, int K, int O) {
  return (size_t)((max_batch + kWgRowsPer - 1) / kWgRowsPer) * (size_t)(K + 1) * O;
}

int dense_wgrad(cudaStream_t s, const float* x, const float* dpred, int B, int K, int O, float* part, float* g) {
  const int np = (B + kWgRowsPer - 1) / kWgRowsPer;
  dense_wgrad_partial<<<dim3((K + 1 + kWgThreads - 1) / kWgThreads, np), kWgThreads, 0, s>>>(x, dpred, B, K, O, part);
  LFMQ_LAUNCH_CHECK();
  const long len = (long)(K + 1) * O;
  dense_wgrad_reduce<<<(unsigned)((len + 255) / 256), 256, 0, s>>>(part, np, len, g);
  LFMQ_LAUNCH_CHECK();
  return 0;
}

}  // namespace lfmq
