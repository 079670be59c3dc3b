// Permutation importance and Shapley attributions (lfmq_chain_permutation_importance, lfmq_chain_shapley): the
// bijection that draws donor windows and group orderings, the kernel that builds the rows of a copy whose high-ranked
// groups come from a donor window, and the fold of a Shapley launch's outputs.  DESIGN.md sections 5e and 5f.
#include "../../include/lfmq.h"
#include "kernels.h"

namespace lfmq {

__host__ __device__ uint32_t perm_index(int32_t N, uint64_t seed, int32_t group, int32_t repeat, uint32_t i) {
  int m = 2;
  while (m < 32 && ((uint64_t)1 << m) < (uint64_t)N) m += 2;
  const int h = m / 2;
  const uint32_t half = ((uint32_t)1 << h) - 1u;
  const uint32_t k0 = (uint32_t)(seed & 0xffffffffu), k1 = (uint32_t)(seed >> 32);
  uint32_t v = i;
  do {        // cycle-walk: 2^m < 4N, so fewer than four passes are expected
    uint32_t L = v >> h, R = v & half;
    for (uint32_t j = 0; j < 4; ++j) {
      uint32_t r[4];
      philox4x32_10(R, j, (uint32_t)group, (uint32_t)repeat, k0, k1, r);
      const uint32_t nR = L ^ (r[0] & half);
      L = R;
      R = nR;
    }
    v = (L << h) | R;
  } while (v >= (uint32_t)N);
  return v;
}

namespace {

constexpr int kPermThreads = 256;
constexpr int kPermRows = 8;      // window rows per CTA: their donors are found once, by one thread each
constexpr int kFoldThreads = 256;

// Rows [a, a + n) of a copy: out[i - a, c] = x[pi(i), c] when rank[col_group[c]] >= k, else x[i, c], with
// pi = perm_index(N, seed, key, rep, .).  Each element reads the one source it needs, and a CTA writes whole rows in
// order, so reads and writes are coalesced.
__global__ void __launch_bounds__(kPermThreads) perm_importance_gather_kernel(
    const float* __restrict__ x, int N, long row_elems, const int32_t* __restrict__ col_group,
    const int32_t* __restrict__ rank, int k, uint64_t seed, int key, int rep, int a, int n, float* __restrict__ out) {
  __shared__ int donor[kPermRows];
  const int i0 = blockIdx.x * kPermRows;
  if (threadIdx.x < kPermRows && i0 + (int)threadIdx.x < n)
    donor[threadIdx.x] = (int)perm_index(N, seed, key, rep, (uint32_t)(a + i0 + threadIdx.x));
  __syncthreads();
  const int rows = min(kPermRows, n - i0);
  for (int j = 0; j < rows; ++j) {
    const float* own = x + (long)(a + i0 + j) * row_elems;
    const float* don = x + (long)donor[j] * row_elems;
    float* dst = out + (long)(i0 + j) * row_elems;
    for (long c = threadIdx.x; c < row_elems; c += kPermThreads)
      dst[c] = (__ldg(rank + __ldg(col_group + c)) >= k ? don : own)[c];
  }
}

// One thread per (window a + i, output o) of a launch of copy (m, k): v = src.p[o][i * stride + off].  k = 0 adds v
// into f_bg; k > 0 adds v - prev into phi[w][o][order[k - 1]], the group copy k adds; k = G also adds v into f_x.
// prev[w][o] = v.  A window's terms arrive in increasing (m, k), one launch after another, so its sums do not depend on
// where launches are cut.  The sums are fp64 and v - prev is exact in fp64: a point model's f_x, M equal forwards over
// M, is its forward bit for bit (an fp32 sum 3v times 1/3 is not v for a third of all v), and sum_g phi telescopes to
// f_x - f_bg before the one rounding to fp32.
__global__ void __launch_bounds__(kFoldThreads) shapley_fold_kernel(
    ShapleySrc src, int K, long stride, long off, int a, int n, int k, int G, const int32_t* __restrict__ order,
    float* __restrict__ prev, double* __restrict__ phi, double* __restrict__ f_x, double* __restrict__ f_bg) {
  const int t = blockIdx.x * kFoldThreads + threadIdx.x;
  if (t >= n * K) return;
  const int i = t / K, o = t - i * K;
  const float* p = src.p[0];
#pragma unroll
  for (int j = 1; j < 2 * LFMQ_MAX_STAGES; ++j)   // selects, not a dynamic index into the parameter array
    if (j == o) p = src.p[j];
  const float v = p[(long)i * stride + off];
  const long wo = (long)(a + i) * K + o;
  if (k == 0) {
    f_bg[wo] += v;
  } else {
    phi[wo * G + order[k - 1]] += (double)v - (double)prev[wo];
    if (k == G) f_x[wo] += v;
  }
  prev[wo] = v;
}

__global__ void shapley_finish_kernel(long n, const double* __restrict__ sum, int samples, float* __restrict__ out) {
  const long j = (long)blockIdx.x * kFoldThreads + threadIdx.x;
  if (j < n) out[j] = (float)(sum[j] / (double)samples);
}

}  // namespace

int perm_importance_gather(cudaStream_t s, const float* x, int N, long row_elems, const int32_t* col_group,
                           const int32_t* rank, int k, uint64_t seed, int key, int rep, int a, int n, float* out) {
  perm_importance_gather_kernel<<<(n + kPermRows - 1) / kPermRows, kPermThreads, 0, s>>>(
      x, N, row_elems, col_group, rank, k, seed, key, rep, a, n, out);
  LFMQ_LAUNCH_CHECK();
  return 0;
}

int shapley_fold(cudaStream_t s, const ShapleySrc& src, int K, long stride, long off, int a, int n, int k, int G,
                 const int32_t* order, float* prev, double* phi, double* f_x, double* f_bg) {
  shapley_fold_kernel<<<(n * K + kFoldThreads - 1) / kFoldThreads, kFoldThreads, 0, s>>>(src, K, stride, off, a, n, k,
                                                                                        G, order, prev, phi, f_x, f_bg);
  LFMQ_LAUNCH_CHECK();
  return 0;
}

int shapley_finish(cudaStream_t s, long n, const double* sum, int samples, float* out) {
  shapley_finish_kernel<<<(unsigned)((n + kFoldThreads - 1) / kFoldThreads), kFoldThreads, 0, s>>>(n, sum, samples,
                                                                                                    out);
  LFMQ_LAUNCH_CHECK();
  return 0;
}

}  // namespace lfmq

extern "C" int32_t lfmq_permutation_index(int32_t N, uint64_t seed, int32_t group, int32_t repeat, int32_t i,
                                          int32_t* out) {
  if (N < 1 || i < 0 || i >= N || group < 0 || repeat < 0 || !out) {
    LFMQ_SET_ERR("lfmq_permutation_index: need N >= 1, 0 <= i < N, group, repeat >= 0 and out (got N %d, i %d, group %d, "
                 "repeat %d)", N, i, group, repeat);
    return LFMQ_ERR_ARG;
  }
  *out = (int32_t)lfmq::perm_index(N, seed, group, repeat, (uint32_t)i);
  return LFMQ_OK;
}
