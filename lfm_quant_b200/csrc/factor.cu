// Lookahead factor backtests (lfmq_factor_eval, DESIGN.md section 5k): each date's rows ranked by each factor score,
// bucketed into Q quantiles, and scored against each outcome measure (bucket means, spread, Spearman IC), with the
// turnover of the top bucket from one date to the next.
//
// order: one radix sort of (date, company) keys gives the base order and the D date segments.  Every score and
// measure is then sorted within the dates by two stable device-wide radix sorts (least significant key first): of
// its order-preserving 64-bit keys (-0 is +0; a non-finite value is the key ~0, which sorts last and drops out) taken
// in base order, then of the dates.  Each segment is in (score, company) order whatever the order of the rows, and
// no sort synchronises with the host.
// ranks: a sorted position i lies in a run [a, b) of equal keys (two binary searches); its average rank is
// (a + b + 1) / 2 and its bucket floor((a + b) Q / 2n) + 1, in integers.  Over the pair set of a factor and a measure
// (the rows where both are finite) the same holds with a and b counted in pair rows: an inclusive scan of the pair
// flags in each sorted order.
// sums: one block per (factor, date) reduces the bucket means (one warp per bucket, lane-strided then a shuffle tree)
// and the centred rank moments of the IC (exact, in 128-bit integers) in segment order, with no atomics.
// turnover: one sort of (company, date) keys gives each row its predecessor at date index d - 1.
#include <cub/device/device_radix_sort.cuh>
#include <cub/device/device_scan.cuh>

#include "../../include/lfmq.h"
#include "kernels.h"

namespace lfmq {
namespace {

constexpr int kThreads = 256;
constexpr int kWarps = kThreads / 32;
constexpr uint64_t kNoKey = ~0ull;

// the order of the doubles as unsigned 64-bit integers; -0 and +0 share a key, non-finite values get kNoKey
__device__ __forceinline__ uint64_t order_key(double v) {
  if (!isfinite(v)) return kNoKey;
  const uint64_t u = (uint64_t)__double_as_longlong(v == 0.0 ? 0.0 : v);
  return (u >> 63) ? ~u : (u | 0x8000000000000000ull);
}

// the first position in [lo, hi) whose key is >= k (<= k for upper_pos), hi if none
__device__ __forceinline__ int lower_pos(const uint64_t* __restrict__ key, int lo, int hi, uint64_t k) {
  while (lo < hi) {
    const int mid = lo + (hi - lo) / 2;
    if (key[mid] < k) lo = mid + 1; else hi = mid;
  }
  return lo;
}

__device__ __forceinline__ int upper_pos(const uint64_t* __restrict__ key, int lo, int hi, uint64_t k) {
  while (lo < hi) {
    const int mid = lo + (hi - lo) / 2;
    if (key[mid] <= k) lo = mid + 1; else hi = mid;
  }
  return lo;
}

// the date segment d (seg_off[d] <= i < seg_off[d + 1]) of a position i < seg_off[D]
__device__ __forceinline__ int segment_of(const int32_t* __restrict__ seg_off, int D, int i) {
  int lo = 0, hi = D;
  while (hi - lo > 1) {
    const int mid = lo + (hi - lo) / 2;
    if (seg_off[mid] <= i) lo = mid; else hi = mid;
  }
  return lo;
}

// the bucket 1..Q of the run [a, b) (positions relative to the segment) among n finite keys
__device__ __forceinline__ int bucket_of(long a, long b, long n, int Q) { return (int)((a + b) * Q / (2 * n)) + 1; }

__device__ __forceinline__ int bucket_at(const uint64_t* __restrict__ key, int s0, int s1, int i, int Q) {
  const uint64_t k = key[i];
  return bucket_of(lower_pos(key, s0, i, k) - s0, upper_pos(key, i + 1, s1, k) - s0, s1 - s0, Q);
}

// key[i] = (date, company) (by_company: (company, date)), idx[i] = i; the company's sign bit is flipped so that the
// codes order as signed integers
__global__ void __launch_bounds__(kThreads) factor_row_keys_kernel(int N, const int32_t* __restrict__ date,
                                                                   const int32_t* __restrict__ company,
                                                                   int by_company, uint64_t* __restrict__ key,
                                                                   int32_t* __restrict__ idx) {
  const int i = blockIdx.x * kThreads + threadIdx.x;
  if (i >= N) return;
  const uint64_t d = (uint32_t)date[i], c = (uint32_t)company[i] ^ 0x80000000u;
  key[i] = by_company ? (c << 32 | d) : (d << 32 | c);
  idx[i] = i;
}

// seg_off[d] = the first base position of date d, d = 0..D
__global__ void __launch_bounds__(kThreads) factor_segments_kernel(int N, int D, const uint64_t* __restrict__ key,
                                                                   int32_t* __restrict__ seg_off) {
  const int d = blockIdx.x * kThreads + threadIdx.x;
  if (d <= D) seg_off[d] = lower_pos(key, 0, N, (uint64_t)d << 32);
}

// pred[row] = the row of the same company at date index d - 1, or -1 (key sorted by (company, date))
__global__ void __launch_bounds__(kThreads) factor_pred_kernel(int N, const uint64_t* __restrict__ key,
                                                               const int32_t* __restrict__ row,
                                                               int32_t* __restrict__ pred) {
  const int i = blockIdx.x * kThreads + threadIdx.x;
  if (i < N) pred[row[i]] = (i > 0 && key[i - 1] + 1 == key[i]) ? row[i - 1] : -1;
}

// the sort input of one score or measure v [N], in base order
__global__ void __launch_bounds__(kThreads) factor_value_keys_kernel(int N, const double* __restrict__ v,
                                                                     const int32_t* __restrict__ base_row,
                                                                     uint64_t* __restrict__ key,
                                                                     int32_t* __restrict__ row) {
  const int i = blockIdx.x * kThreads + threadIdx.x;
  if (i >= N) return;
  const int r = base_row[i];
  key[i] = order_key(v[r]);
  row[i] = r;
}

// d[i] = the date of the row at sorted position i, idx[i] = i
__global__ void __launch_bounds__(kThreads) factor_date_keys_kernel(int N, const int32_t* __restrict__ date,
                                                                    const int32_t* __restrict__ row,
                                                                    uint32_t* __restrict__ d,
                                                                    int32_t* __restrict__ idx) {
  const int i = blockIdx.x * kThreads + threadIdx.x;
  if (i >= N) return;
  d[i] = (uint32_t)date[row[i]];
  idx[i] = i;
}

// key / row [j] = skey / srow [pos[j]]
__global__ void __launch_bounds__(kThreads) factor_gather_kernel(int N, const int32_t* __restrict__ pos,
                                                                 const uint64_t* __restrict__ skey,
                                                                 const int32_t* __restrict__ srow,
                                                                 uint64_t* __restrict__ key,
                                                                 int32_t* __restrict__ row) {
  const int j = blockIdx.x * kThreads + threadIdx.x;
  if (j >= N) return;
  const int p = pos[j];
  key[j] = skey[p];
  row[j] = srow[p];
}

// bq[row] = the bucket 1..Q of every row with a finite score (rows without keep the 0 they were cleared to)
__global__ void __launch_bounds__(kThreads) factor_bucket_kernel(int D, int Q, const int32_t* __restrict__ seg_off,
                                                                 const uint64_t* __restrict__ key,
                                                                 const int32_t* __restrict__ row,
                                                                 uint8_t* __restrict__ bq) {
  const int i = blockIdx.x * kThreads + threadIdx.x;
  if (i >= seg_off[D] || key[i] == kNoKey) return;
  const int d = segment_of(seg_off, D, i);
  const int s0 = seg_off[d];
  const int s1 = lower_pos(key, i, seg_off[d + 1], kNoKey);
  bq[row[i]] = (uint8_t)bucket_at(key, s0, s1, i, Q);
}

// flag[i] = 1 where the sorted position i is a pair row (its key and other[row[i]] finite)
__global__ void __launch_bounds__(kThreads) factor_pair_flags_kernel(int N, const int32_t* __restrict__ seg_end,
                                                                     const uint64_t* __restrict__ key,
                                                                     const int32_t* __restrict__ row,
                                                                     const double* __restrict__ other,
                                                                     int32_t* __restrict__ flag) {
  const int i = blockIdx.x * kThreads + threadIdx.x;
  if (i < N) flag[i] = i < *seg_end && key[i] != kNoKey && isfinite(other[row[i]]);
}

// twice the average rank among the pair rows of its date, of every pair row (pc: the exclusive counts of pair rows,
// pc[i] before position i)
__global__ void __launch_bounds__(kThreads) factor_pair_rank_kernel(int D, const int32_t* __restrict__ seg_off,
                                                                    const uint64_t* __restrict__ key,
                                                                    const int32_t* __restrict__ row,
                                                                    const int32_t* __restrict__ flag,
                                                                    const int32_t* __restrict__ pc,
                                                                    uint32_t* __restrict__ rank2) {
  const int i = blockIdx.x * kThreads + threadIdx.x;
  if (i >= seg_off[D] || !flag[i]) return;
  const int d = segment_of(seg_off, D, i);
  const int s0 = seg_off[d], s1 = seg_off[d + 1];
  const uint64_t k = key[i];
  const long a = pc[lower_pos(key, s0, i, k)] - pc[s0], b = pc[upper_pos(key, i + 1, s1, k)] - pc[s0];
  rank2[row[i]] = (uint32_t)(a + b + 1);
}

template <typename T>
__device__ T block_sum(T v, T* sh) {
  sh[threadIdx.x] = v;
  __syncthreads();
  for (int s = kThreads / 2; s > 0; s >>= 1) {
    if (threadIdx.x < s) sh[threadIdx.x] += sh[threadIdx.x + s];
    __syncthreads();
  }
  const T r = sh[0];
  __syncthreads();
  return r;
}

// One block per date d of factor g: n, bucket_n, turnover, and for every measure the bucket means, spread, n_pair and
// ic.  key / row: the factor's sorted keys and rows; pc [M][N + 1] its pair-row counts per measure; yr [M][N] twice each
// pair row's average measure rank.
__global__ void __launch_bounds__(kThreads) factor_segment_kernel(int N, int D, int M, int Q, int g,
                                                                  const int32_t* __restrict__ seg_off,
                                                                  const uint64_t* __restrict__ key,
                                                                  const int32_t* __restrict__ row,
                                                                  const uint8_t* __restrict__ bq,
                                                                  const int32_t* __restrict__ pred,
                                                                  const double* __restrict__ measure,
                                                                  const int32_t* __restrict__ pcg,
                                                                  const uint32_t* __restrict__ yr, FactorOut o) {
  __shared__ int lo[LFMQ_FACTOR_MAX_Q + 1];          // bucket q is [lo[q - 1], lo[q])
  __shared__ double mean[LFMQ_FACTOR_MAX_Q];
  __shared__ long long red_n[kThreads];
  __shared__ __int128 red_m[kThreads];
  const int d = blockIdx.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int s0 = seg_off[d], s1 = seg_off[d + 1];
  const int e = lower_pos(key, s0, s1, kNoKey), n = e - s0;    // the finite scores are [s0, e)
  for (int q = tid; q <= Q; q += kThreads) {
    int a = s0, b = e;                                           // the first position whose bucket exceeds q
    if (q == 0) b = s0;
    else if (q < Q)
      while (a < b) {
        const int mid = a + (b - a) / 2;
        if (bucket_at(key, s0, e, mid, Q) <= q) a = mid + 1; else b = mid;
      }
    lo[q] = b;
  }
  __syncthreads();
  const long gd = (long)g * D + d;
  if (tid == 0) o.n[gd] = n;
  for (int q = tid; q < Q; q += kThreads) o.bucket_n[gd * Q + q] = lo[q + 1] - lo[q];
  long long fresh = 0;                                           // top-bucket rows not in the top bucket at d - 1
  for (int i = lo[Q - 1] + tid; i < lo[Q]; i += kThreads) {
    const int p = pred[row[i]];
    fresh += p < 0 || bq[p] != Q;
  }
  fresh = block_sum(fresh, red_n);
  if (tid == 0) {
    const int top = lo[Q] - lo[Q - 1];
    o.turnover[gd] = (d == 0 || top == 0) ? (double)NAN : (double)fresh / (double)top;
  }
  for (int m = 0; m < M; ++m) {
    const double* mv = measure + (long)m * N;
    const long gmd = ((long)g * M + m) * D + d;
    for (int q = warp; q < Q; q += kWarps) {
      double sum = 0.0;
      int cnt = 0;
      for (int i = lo[q] + lane; i < lo[q + 1]; i += 32) {
        const double v = mv[row[i]];
        if (isfinite(v)) {
          sum += v;
          ++cnt;
        }
      }
      for (int off = 16; off > 0; off >>= 1) {
        sum += __shfl_down_sync(0xffffffffu, sum, off);
        cnt += __shfl_down_sync(0xffffffffu, cnt, off);
      }
      if (lane == 0) {
        mean[q] = cnt ? sum / (double)cnt : (double)NAN;
        o.bucket_mean[gmd * Q + q] = mean[q];
      }
    }
    // Spearman: the Pearson correlation of the pair ranks, from exact sums of the centred doubled ranks 2r - (np + 1)
    const int32_t* pc = pcg + (long)m * (N + 1);
    const uint32_t* y2 = yr + (long)m * N;
    const long np = pc[s1] - pc[s0], c = np + 1;
    __int128 sxy = 0, sxx = 0, syy = 0;
    for (int i = s0 + tid; i < e; i += kThreads) {
      const int r = row[i];
      if (!isfinite(mv[r])) continue;
      const uint64_t k = key[i];
      const long x = (long)(pc[lower_pos(key, s0, i, k)] - pc[s0]) + (pc[upper_pos(key, i + 1, e, k)] - pc[s0]) + 1 - c;
      const long y = (long)y2[r] - c;
      sxy += (__int128)x * y;
      sxx += (__int128)x * x;
      syy += (__int128)y * y;
    }
    sxy = block_sum(sxy, red_m);
    sxx = block_sum(sxx, red_m);
    syy = block_sum(syy, red_m);
    if (tid == 0) {
      o.n_pair[gmd] = (int32_t)np;
      o.ic[gmd] = (np < 3 || sxx == 0 || syy == 0) ? (double)NAN
                                                     : (double)sxy / sqrt((double)sxx * (double)syy);
      o.spread[gmd] = mean[Q - 1] - mean[0];
    }
    __syncthreads();
  }
}

#define RUN_FACTOR(expr)   \
  do {                     \
    const int _rc = (expr); \
    if (_rc != 0) return _rc; \
  } while (0)

inline unsigned blocks(long n) { return (unsigned)((n + kThreads - 1) / kThreads); }

int date_bits(int D) {
  int b = 0;
  while ((1L << b) < D) ++b;
  return b;
}

// key / row [N]: the values v [N] of every row, sorted within the dates in (date, key, company) order.  DeviceRadixSort
// is stable, so sorting the keys taken in base (date, company) order and then the dates leaves equal keys of one date
// in company order.
int sort_within_dates(cudaStream_t s, int N, int D, const int32_t* date, const double* v, const FactorWork& w,
                      size_t temp_bytes, uint64_t* key, int32_t* row) {
  factor_value_keys_kernel<<<blocks(N), kThreads, 0, s>>>(N, v, w.base_row, w.k0, w.v0);
  LFMQ_LAUNCH_CHECK();
  LFMQ_CUDA_CHECK(cub::DeviceRadixSort::SortPairs(w.temp, temp_bytes, w.k0, w.k1, w.v0, w.v1, N, 0, 64, s));
  factor_date_keys_kernel<<<blocks(N), kThreads, 0, s>>>(N, date, w.v1, w.d0, w.v0);
  LFMQ_LAUNCH_CHECK();
  LFMQ_CUDA_CHECK(cub::DeviceRadixSort::SortPairs(w.temp, temp_bytes, w.d0, w.d1, w.v0, w.pos, N, 0,
                                                  std::max(1, date_bits(D)), s));
  factor_gather_kernel<<<blocks(N), kThreads, 0, s>>>(N, w.pos, w.k1, w.v1, key, row);
  LFMQ_LAUNCH_CHECK();
  return 0;
}

}  // namespace

int factor_temp_bytes(int N, int D, size_t* bytes) {
  size_t a = 0, b = 0, c = 0;
  LFMQ_CUDA_CHECK(cub::DeviceRadixSort::SortPairs(nullptr, a, (const uint64_t*)nullptr, (uint64_t*)nullptr,
                                                  (const int32_t*)nullptr, (int32_t*)nullptr, N, 0, 64));
  LFMQ_CUDA_CHECK(cub::DeviceRadixSort::SortPairs(nullptr, b, (const uint32_t*)nullptr, (uint32_t*)nullptr,
                                                  (const int32_t*)nullptr, (int32_t*)nullptr, N, 0,
                                                  std::max(1, date_bits(D))));
  LFMQ_CUDA_CHECK(cub::DeviceScan::InclusiveSum(nullptr, c, (const int32_t*)nullptr, (int32_t*)nullptr, N));
  *bytes = std::max(a, std::max(b, c));
  return 0;
}

int factor_eval(cudaStream_t s, const int32_t* date, const int32_t* company, int N, int D, const double* score, int G,
                const double* measure, int M, int Q, const FactorWork& w, size_t temp_bytes, FactorOut o) {
  // base order (date, company) and the date segments
  factor_row_keys_kernel<<<blocks(N), kThreads, 0, s>>>(N, date, company, 0, w.k0, w.v0);
  LFMQ_LAUNCH_CHECK();
  LFMQ_CUDA_CHECK(cub::DeviceRadixSort::SortPairs(w.temp, temp_bytes, w.k0, w.k1, w.v0, w.base_row, N, 0,
                                                  32 + date_bits(D), s));
  factor_segments_kernel<<<blocks((long)D + 1), kThreads, 0, s>>>(N, D, w.k1, w.seg_off);
  LFMQ_LAUNCH_CHECK();
  // each row's predecessor at date index d - 1
  factor_row_keys_kernel<<<blocks(N), kThreads, 0, s>>>(N, date, company, 1, w.k0, w.v0);
  LFMQ_LAUNCH_CHECK();
  LFMQ_CUDA_CHECK(cub::DeviceRadixSort::SortPairs(w.temp, temp_bytes, w.k0, w.k1, w.v0, w.v1, N, 0, 64, s));
  factor_pred_kernel<<<blocks(N), kThreads, 0, s>>>(N, w.k1, w.v1, w.pred);
  LFMQ_LAUNCH_CHECK();
  // every measure sorted within the dates
  for (int m = 0; m < M; ++m) {
    RUN_FACTOR(sort_within_dates(s, N, D, date, measure + (long)m * N, w, temp_bytes, w.mkey + (long)m * N,
                                 w.mrow + (long)m * N));
  }
  for (int g = 0; g < G; ++g) {
    const double* sg = score + (long)g * N;
    RUN_FACTOR(sort_within_dates(s, N, D, date, sg, w, temp_bytes, w.gkey, w.grow));
    LFMQ_CUDA_CHECK(cudaMemsetAsync(w.bq, 0, (size_t)N, s));
    factor_bucket_kernel<<<blocks(N), kThreads, 0, s>>>(D, Q, w.seg_off, w.gkey, w.grow, w.bq);
    LFMQ_LAUNCH_CHECK();
    for (int m = 0; m < M; ++m) {
      int32_t* pcg = w.pcg + (long)m * (N + 1);
      const uint64_t* mkey = w.mkey + (long)m * N;
      const int32_t* mrow = w.mrow + (long)m * N;
      // pair counts in the factor's order, then in the measure's order and the measure ranks of the pair rows
      factor_pair_flags_kernel<<<blocks(N), kThreads, 0, s>>>(N, w.seg_off + D, w.gkey, w.grow, measure + (long)m * N,
                                                              w.flag);
      LFMQ_LAUNCH_CHECK();
      LFMQ_CUDA_CHECK(cudaMemsetAsync(pcg, 0, sizeof(int32_t), s));
      LFMQ_CUDA_CHECK(cub::DeviceScan::InclusiveSum(w.temp, temp_bytes, w.flag, pcg + 1, N, s));
      factor_pair_flags_kernel<<<blocks(N), kThreads, 0, s>>>(N, w.seg_off + D, mkey, mrow, sg, w.flag);
      LFMQ_LAUNCH_CHECK();
      LFMQ_CUDA_CHECK(cudaMemsetAsync(w.pcm, 0, sizeof(int32_t), s));
      LFMQ_CUDA_CHECK(cub::DeviceScan::InclusiveSum(w.temp, temp_bytes, w.flag, w.pcm + 1, N, s));
      factor_pair_rank_kernel<<<blocks(N), kThreads, 0, s>>>(D, w.seg_off, mkey, mrow, w.flag, w.pcm,
                                                             w.yr + (long)m * N);
      LFMQ_LAUNCH_CHECK();
    }
    factor_segment_kernel<<<D, kThreads, 0, s>>>(N, D, M, Q, g, w.seg_off, w.gkey, w.grow, w.bq, w.pred, measure,
                                                 w.pcg, w.yr, o);
    LFMQ_LAUNCH_CHECK();
  }
  return 0;
}

}  // namespace lfmq
