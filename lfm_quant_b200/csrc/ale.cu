// Accumulated local effects (lfmq_chain_ale): the per-feature sort of the windows' values with its edges and bins, the
// kernel that builds the rows of a copy whose one column sits at its bin's lower or upper edge, the pick of each
// window's local effect and the fold of those effects over the bins.  DESIGN.md section 5h.
#include <algorithm>

#include <cub/device/device_segmented_radix_sort.cuh>

#include "../../include/lfmq.h"
#include "kernels.h"

namespace lfmq {

namespace {

constexpr int kKeyThreads = 256;
constexpr int kEdgeThreads = 256;
constexpr int kGatherThreads = 256;
constexpr int kGatherRows = 8;
constexpr int kPickThreads = 256;
constexpr int kFoldThreads = 256;

// key [g][i] = x[i, cols[g]] (+0 for -0, +inf for a non-finite value, so that the finite values sort first), val = i;
// off [g] = g * N for g <= G: the segments of the sort.
__global__ void __launch_bounds__(kKeyThreads) ale_keys_kernel(const float* __restrict__ x, int N, long row_elems,
                                                               const int32_t* __restrict__ cols, int G,
                                                               float* __restrict__ key, int32_t* __restrict__ val,
                                                               int32_t* __restrict__ off) {
  const long t = (long)blockIdx.x * kKeyThreads + threadIdx.x;
  if (t <= G) off[t] = (int32_t)(t * N);
  if (t >= (long)G * N) return;
  const int g = (int)(t / N), i = (int)(t - (long)g * N);
  const float v = x[(long)i * row_elems + cols[g]];
  key[t] = isfinite(v) ? v + 0.0f : INFINITY;
  val[t] = i;
}

// One CTA per feature g over its sorted values s [N] (the window of s[p] is w[p]).  N' = the finite values; the
// type-1 quantiles q_0 = s[0], q_k = s[ceil(k N' / K) - 1] with repeats dropped are the edges z_0 < .. < z_Kg; e_k = the
// finite values <= z_k, so bin k (1-based) is the sorted run [e_{k-1}, e_k) with e_0 = 0.  Writes edges [K+1] (NaN past
// Kg, and at 0 when N' = 0), counts [K], ends [K+1] = e, n_bins = Kg and bin_of [N] = each window's bin (0: none).
__global__ void __launch_bounds__(kEdgeThreads) ale_edges_kernel(const float* __restrict__ skey,
                                                                 const int32_t* __restrict__ sval, int N, int K,
                                                                 int32_t* __restrict__ n_bins, float* __restrict__ edges,
                                                                 int32_t* __restrict__ counts,
                                                                 int32_t* __restrict__ ends,
                                                                 int32_t* __restrict__ bin_of) {
  __shared__ float z[LFMQ_ALE_MAX_BINS + 1];
  __shared__ int32_t e[LFMQ_ALE_MAX_BINS + 1];
  __shared__ int nz;
  const int g = blockIdx.x;
  const float* s = skey + (long)g * N;
  const int32_t* w = sval + (long)g * N;
  float* ed = edges + (long)g * (K + 1);
  int32_t* ct = counts + (long)g * K;
  int32_t* en = ends + (long)g * (K + 1);
  int32_t* bo = bin_of + (long)g * N;
  if (threadIdx.x == 0) {
    int lo = 0, hi = N;                                   // N' = the first +inf
    while (lo < hi) {
      const int mid = (lo + hi) / 2;
      if (s[mid] < INFINITY) lo = mid + 1; else hi = mid;
    }
    const int nf = lo;
    int m = 0;
    if (nf > 0) {
      z[m++] = s[0];
      for (int k = 1; k <= K; ++k) {
        const float v = s[((int64_t)k * nf + K - 1) / K - 1];
        if (v > z[m - 1]) z[m++] = v;
      }
    }
    nz = m;
  }
  __syncthreads();
  const int Kg = nz > 1 ? nz - 1 : 0;
  for (int k = threadIdx.x; k <= K; k += kEdgeThreads) {
    ed[k] = k < nz ? z[k] : NAN;
    int ek = 0;
    if (k <= Kg && Kg > 0) {
      int lo = 0, hi = N;                                 // the values <= z_k
      while (lo < hi) {
        const int mid = (lo + hi) / 2;
        if (s[mid] <= z[k]) lo = mid + 1; else hi = mid;
      }
      ek = lo;
    }
    e[k] = ek;
    en[k] = ek;
  }
  __syncthreads();
  for (int k = 1 + threadIdx.x; k <= K; k += kEdgeThreads) ct[k - 1] = k <= Kg ? e[k] - (k == 1 ? 0 : e[k - 1]) : 0;
  if (threadIdx.x == 0) n_bins[g] = Kg;
  const int nf = Kg > 0 ? e[Kg] : 0;
  for (int p = threadIdx.x; p < N; p += kEdgeThreads) {
    int b = 0;
    if (p < nf) {                                         // the first k >= 1 with p < e_k
      int lo = 1, hi = Kg;
      while (lo < hi) {
        const int mid = (lo + hi) / 2;
        if (p < e[mid]) hi = mid; else lo = mid + 1;
      }
      b = lo;
    }
    bo[w[p]] = b;
  }
}

// Rows [a, a + n) of a copy: out[i - a] = x[i] with column `col` set to edge[bin_of[i] - 1 + upper] (x's own value for a
// window without a bin).  A CTA writes whole rows in order, so reads and writes are coalesced.
__global__ void __launch_bounds__(kGatherThreads) ale_gather_kernel(const float* __restrict__ x, long row_elems,
                                                                    int col, const int32_t* __restrict__ bin_of,
                                                                    const float* __restrict__ edge, int upper, int a,
                                                                    int n, float* __restrict__ out) {
  const int i0 = blockIdx.x * kGatherRows;
  const int rows = min(kGatherRows, n - i0);
  for (int j = 0; j < rows; ++j) {
    const int b = __ldg(bin_of + a + i0 + j);
    const float* src = x + (long)(a + i0 + j) * row_elems;
    float* dst = out + (long)(i0 + j) * row_elems;
    for (long c = threadIdx.x; c < row_elems; c += kGatherThreads)
      dst[c] = (c == col && b > 0) ? __ldg(edge + b - 1 + upper) : src[c];
  }
}

// One thread per (window a + i, output o) of a launch: v = src.p[o][i * stride + off]; d[a + i][o] = v on the upper
// copy, d[a + i][o] -= v on the lower one, so that d holds f(upper) - f(lower) in fp32.
__global__ void __launch_bounds__(kPickThreads) ale_pick_kernel(ShapleySrc src, int J, long stride, long off, int a,
                                                                int n, int upper, float* __restrict__ d) {
  const int t = blockIdx.x * kPickThreads + threadIdx.x;
  if (t >= n * J) return;
  const int i = t / J, o = t - i * J;
  const float* p = src.p[0];
#pragma unroll
  for (int j = 1; j < 2 * LFMQ_MAX_STAGES; ++j)   // selects, not a dynamic index into the parameter array
    if (j == o) p = src.p[j];
  const float v = p[(long)i * stride + off];
  float* dst = d + (long)(a + i) * J + o;
  *dst = upper ? v : *dst - v;
}

// One CTA for feature g.  Warp-strided over the (bin, output) pairs: each lane sums d over its share of the bin's sorted
// run in fp64, a fixed xor-shuffle tree adds the lanes, and a second pass gives the population variance about the mean.
// Then one thread per output runs the prefix sum g(z_k) and the centring of ALEPlot in fp64.  No atomics: the results
// depend only on d and the sorted order.
__global__ void __launch_bounds__(kFoldThreads) ale_fold_kernel(const int32_t* __restrict__ sval,
                                                                const int32_t* __restrict__ ends, const int32_t* n_bins,
                                                                int g, int N, int K, int J,
                                                                const float* __restrict__ d, double* __restrict__ mean,
                                                                float* __restrict__ ale, float* __restrict__ local_mean,
                                                                float* __restrict__ local_sd) {
  const int Kg = n_bins[g];
  const int32_t* w = sval + (long)g * N;
  const int32_t* e = ends + (long)g * (K + 1);
  float* al = ale + (long)g * (K + 1) * J;
  float* lm = local_mean + (long)g * K * J;
  float* ls = local_sd + (long)g * K * J;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  for (int q = warp; q < Kg * J; q += kFoldThreads / 32) {
    const int k = q / J, o = q - k * J;                   // bin k + 1
    const int p0 = k == 0 ? 0 : e[k], p1 = e[k + 1];
    double s = 0.0;
    for (int p = p0 + lane; p < p1; p += 32) s += (double)d[(long)w[p] * J + o];
    for (int m = 16; m > 0; m >>= 1) s += __shfl_xor_sync(0xffffffffu, s, m);
    const double mu = s / (double)(p1 - p0);
    double v = 0.0;
    for (int p = p0 + lane; p < p1; p += 32) {
      const double r = (double)d[(long)w[p] * J + o] - mu;
      v += r * r;
    }
    for (int m = 16; m > 0; m >>= 1) v += __shfl_xor_sync(0xffffffffu, v, m);
    if (lane == 0) {
      mean[q] = mu;
      lm[q] = (float)mu;
      ls[q] = (float)sqrt(v / (double)(p1 - p0));
    }
  }
  for (int q = Kg * J + threadIdx.x; q < K * J; q += kFoldThreads) lm[q] = ls[q] = NAN;
  __syncthreads();
  for (int o = threadIdx.x; o < J; o += kFoldThreads) {
    if (Kg == 0) {
      for (int k = 0; k <= K; ++k) al[(long)k * J + o] = NAN;
      continue;
    }
    double acc = 0.0, c = 0.0;                            // c = sum_k n_k (g(z_{k-1}) + g(z_k)) / 2
    for (int k = 1; k <= Kg; ++k) {
      const double prev = acc;
      acc += mean[(long)(k - 1) * J + o];
      c += (double)(e[k] - (k == 1 ? 0 : e[k - 1])) * 0.5 * (prev + acc);
    }
    c /= (double)e[Kg];
    acc = 0.0;
    al[o] = (float)(0.0 - c);
    for (int k = 1; k <= K; ++k) {
      if (k <= Kg) acc += mean[(long)(k - 1) * J + o];
      al[(long)k * J + o] = k <= Kg ? (float)(acc - c) : NAN;
    }
  }
}

}  // namespace

int ale_sort_bytes(int N, int G, size_t* bytes) {
  *bytes = 0;
  LFMQ_CUDA_CHECK(cub::DeviceSegmentedRadixSort::SortPairs(nullptr, *bytes, (const float*)nullptr, (float*)nullptr,
                                                           (const int32_t*)nullptr, (int32_t*)nullptr, N * G, G,
                                                           (const int32_t*)nullptr, (const int32_t*)nullptr));
  return 0;
}

int ale_bins(cudaStream_t s, const float* x, int N, long row_elems, const int32_t* cols, int G, int K, void* temp,
             size_t temp_bytes, const AleSort& w, int32_t* n_bins, float* edges, int32_t* counts) {
  const long n = (long)G * N;
  ale_keys_kernel<<<(unsigned)((std::max<long>(n, G + 1) + kKeyThreads - 1) / kKeyThreads), kKeyThreads, 0, s>>>(
      x, N, row_elems, cols, G, w.key, w.val, w.off);
  LFMQ_LAUNCH_CHECK();
  LFMQ_CUDA_CHECK(cub::DeviceSegmentedRadixSort::SortPairs(temp, temp_bytes, w.key, w.skey, w.val, w.sval, (int)n, G,
                                                           w.off, w.off + 1, 0, 32, s));
  ale_edges_kernel<<<G, kEdgeThreads, 0, s>>>(w.skey, w.sval, N, K, n_bins, edges, counts, w.ends, w.bin_of);
  LFMQ_LAUNCH_CHECK();
  return 0;
}

int ale_gather(cudaStream_t s, const float* x, long row_elems, int col, const int32_t* bin_of, const float* edge,
               int upper, int a, int n, float* out) {
  ale_gather_kernel<<<(n + kGatherRows - 1) / kGatherRows, kGatherThreads, 0, s>>>(x, row_elems, col, bin_of, edge,
                                                                                   upper, a, n, out);
  LFMQ_LAUNCH_CHECK();
  return 0;
}

int ale_pick(cudaStream_t s, const ShapleySrc& src, int J, long stride, long off, int a, int n, int upper, float* d) {
  ale_pick_kernel<<<(n * J + kPickThreads - 1) / kPickThreads, kPickThreads, 0, s>>>(src, J, stride, off, a, n, upper,
                                                                                    d);
  LFMQ_LAUNCH_CHECK();
  return 0;
}

int ale_fold(cudaStream_t s, const AleSort& w, const int32_t* n_bins, int g, int N, int K, int J, const float* d,
             double* mean, float* ale, float* local_mean, float* local_sd) {
  ale_fold_kernel<<<1, kFoldThreads, 0, s>>>(w.sval, w.ends, n_bins, g, N, K, J, d, mean, ale, local_mean, local_sd);
  LFMQ_LAUNCH_CHECK();
  return 0;
}

}  // namespace lfmq
