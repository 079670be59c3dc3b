// Split-conformal prediction intervals (lfmq_conformal_*, DESIGN.md section 5j): the nonconformity scores of a set of
// windows, the per-step sort of the calibration scores with the rank rule that picks q_hat, and the intervals and
// p-values of the query windows.
//
// score: r = |y - pred| (/ scale), in IEEE single precision with no contraction (__fsub_rn, __fdiv_rn), so that it is
// the bits NumPy's float32 arithmetic gives; NaN (0x7fffffff) where y is not finite.
// sort: scores are >= 0 or NaN, so their bits order like their values, NaN last.  The key (s << 32 | bits(r)) sorts
// every step's scores in one device-wide radix sort; step s's sorted run is keys [s * Nc, (s + 1) * Nc).
// select: n = the scores before the first NaN; q_hat[s][k] = sorted[s][ceil((n + 1) l_k) - 1], +inf past n.
// apply: lower / upper = pred -/+ q_hat * scale (each rounded once), one thread per element; p = (1 + #{r_i >= r}) /
// (n + 1) by binary search, one thread per window.
#include <cub/device/device_radix_sort.cuh>

#include "../../include/lfmq.h"
#include "kernels.h"

namespace lfmq {
namespace {

constexpr int kThreads = 256;

__device__ __forceinline__ float conf_score(float p, float y, const float* __restrict__ scale, long i) {
  if (!isfinite(y)) return __int_as_float(0x7fffffff);
  float r = fabsf(__fsub_rn(y, p));
  if (scale) r = __fdiv_rn(r, scale[i]);
  return r != r ? __int_as_float(0x7fffffff) : r;
}

__global__ void __launch_bounds__(kThreads) conformal_score_kernel(long n, const float* __restrict__ pred,
                                                                   const float* __restrict__ y,
                                                                   const float* __restrict__ scale,
                                                                   float* __restrict__ r) {
  const long i = (long)blockIdx.x * kThreads + threadIdx.x;
  if (i < n) r[i] = conf_score(pred[i], y[i], scale, i);
}

// key[s * Nc + i] = (s << 32) | bits(r[s][i])
__global__ void __launch_bounds__(kThreads) conformal_keys_kernel(int S, int Nc, const float* __restrict__ pred,
                                                                  const float* __restrict__ y,
                                                                  const float* __restrict__ scale,
                                                                  uint64_t* __restrict__ key) {
  const long i = (long)blockIdx.x * kThreads + threadIdx.x;
  if (i >= (long)S * Nc) return;
  const uint64_t s = (uint64_t)(i / Nc);
  key[i] = (s << 32) | (uint64_t)__float_as_uint(conf_score(pred[i], y[i], scale, i));
}

__global__ void __launch_bounds__(kThreads) conformal_unkey_kernel(long n, const uint64_t* __restrict__ key,
                                                                   float* __restrict__ sorted) {
  const long i = (long)blockIdx.x * kThreads + threadIdx.x;
  if (i < n) sorted[i] = __uint_as_float((uint32_t)(key[i] & 0xffffffffu));
}

struct Levels {
  double l[LFMQ_CONFORMAL_MAX_LEVELS];
};

// One warp per step s: n_valid[s] and q_hat[s][Q].
__global__ void conformal_select_kernel(int Nc, int Q, Levels lv, const float* __restrict__ sorted,
                                        int32_t* __restrict__ n_valid, float* __restrict__ qhat) {
  const int s = blockIdx.x;
  const float* v = sorted + (long)s * Nc;
  int lo = 0, hi = Nc;                       // the first NaN
  while (lo < hi) {
    const int mid = (lo + hi) / 2;
    if (v[mid] == v[mid]) lo = mid + 1; else hi = mid;
  }
  const int n = lo;
  if (threadIdx.x == 0) n_valid[s] = n;
  for (int k = threadIdx.x; k < Q; k += blockDim.x) {
    const double rank = ceil((double)(n + 1) * lv.l[k]);
    qhat[(long)s * Q + k] = rank <= (double)n ? v[(long)rank - 1] : INFINITY;
  }
}

// One thread per element (s, i, k) of the bounds, so that the stores of a warp are contiguous.
__global__ void __launch_bounds__(kThreads) conformal_bounds_kernel(int S, int N, int Q,
                                                                    const float* __restrict__ pred,
                                                                    const float* __restrict__ scale,
                                                                    const float* __restrict__ qhat,
                                                                    float* __restrict__ lower,
                                                                    float* __restrict__ upper) {
  const long e = (long)blockIdx.x * kThreads + threadIdx.x;
  if (e >= (long)S * N * Q) return;
  const long i = e / Q;                      // s * N + window
  const int k = (int)(e - i * Q), s = (int)(i / N);
  const float p = pred[i];
  const float w = __fmul_rn(qhat[(long)s * Q + k], scale ? scale[i] : 1.f);
  lower[e] = __fsub_rn(p, w);
  upper[e] = __fadd_rn(p, w);
}

// One thread per (s, i) of the query windows: the p-value by binary search in step s's sorted scores.
__global__ void __launch_bounds__(kThreads) conformal_pvalue_kernel(int S, int N, int Nc,
                                                                    const float* __restrict__ pred,
                                                                    const float* __restrict__ y,
                                                                    const float* __restrict__ scale,
                                                                    const float* __restrict__ sorted,
                                                                    const int32_t* __restrict__ n_valid,
                                                                    float* __restrict__ pvalue) {
  const long i = (long)blockIdx.x * kThreads + threadIdx.x;
  if (i >= (long)S * N) return;
  const int s = (int)(i / N);
  float pv = __int_as_float(0x7fffffff);
  if (y) {
    const float r = conf_score(pred[i], y[i], scale, i);
    if (r == r) {
      const int n = n_valid[s];
      const float* v = sorted + (long)s * Nc;
      int lo = 0, hi = n;                    // the first score >= r
      while (lo < hi) {
        const int mid = (lo + hi) / 2;
        if (v[mid] < r) lo = mid + 1; else hi = mid;
      }
      pv = __fdiv_rn((float)(1 + n - lo), (float)(n + 1));
    }
  }
  pvalue[i] = pv;
}

inline unsigned blocks(long n) { return (unsigned)((n + kThreads - 1) / kThreads); }

// the bits of the sort key: 32 for the score, enough above them for the step
inline int key_bits(int S) {
  int b = 0;
  while ((1 << b) < S) ++b;
  return 32 + b;
}

}  // namespace

int conformal_sort_bytes(int S, int Nc, size_t* bytes) {
  *bytes = 0;
  LFMQ_CUDA_CHECK(cub::DeviceRadixSort::SortKeys(nullptr, *bytes, (const uint64_t*)nullptr, (uint64_t*)nullptr,
                                                 (int)((long)S * Nc), 0, key_bits(S)));
  return 0;
}

int conformal_scores(cudaStream_t s, long n, const float* pred, const float* y, const float* scale, float* r) {
  conformal_score_kernel<<<blocks(n), kThreads, 0, s>>>(n, pred, y, scale, r);
  LFMQ_LAUNCH_CHECK();
  return 0;
}

int conformal_calibrate(cudaStream_t s, int S, int Nc, const float* pred, const float* y, const float* scale,
                        const double* levels, int Q, void* temp, size_t temp_bytes, uint64_t* key, uint64_t* skey,
                        int32_t* n_valid, float* sorted, float* qhat) {
  const long n = (long)S * Nc;
  conformal_keys_kernel<<<blocks(n), kThreads, 0, s>>>(S, Nc, pred, y, scale, key);
  LFMQ_LAUNCH_CHECK();
  LFMQ_CUDA_CHECK(cub::DeviceRadixSort::SortKeys(temp, temp_bytes, key, skey, (int)n, 0, key_bits(S), s));
  conformal_unkey_kernel<<<blocks(n), kThreads, 0, s>>>(n, skey, sorted);
  LFMQ_LAUNCH_CHECK();
  Levels lv{};
  for (int k = 0; k < Q; ++k) lv.l[k] = levels[k];
  conformal_select_kernel<<<S, 32, 0, s>>>(Nc, Q, lv, sorted, n_valid, qhat);
  LFMQ_LAUNCH_CHECK();
  return 0;
}

int conformal_apply(cudaStream_t s, int S, int N, int Nc, int Q, const float* pred, const float* y, const float* scale,
                    const float* sorted, const int32_t* n_valid, const float* qhat, float* lower, float* upper,
                    float* pvalue) {
  conformal_bounds_kernel<<<blocks((long)S * N * Q), kThreads, 0, s>>>(S, N, Q, pred, scale, qhat, lower, upper);
  LFMQ_LAUNCH_CHECK();
  conformal_pvalue_kernel<<<blocks((long)S * N), kThreads, 0, s>>>(S, N, Nc, pred, y, scale, sorted, n_valid, pvalue);
  LFMQ_LAUNCH_CHECK();
  return 0;
}

}  // namespace lfmq
