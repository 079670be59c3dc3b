// Permutation importance (lfmq_chain_permutation_importance): the bijection that shuffles one group of input columns
// across the held-out windows, and the kernel that builds the rows of a permuted copy.  DESIGN.md section 5e.
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

// Rows [a, a + n) of copy (g, r): out[i - a, c] = x[pi(i), c] when col_group[c] == g, else x[i, c].  Each element reads
// the one source it needs, and a CTA writes whole rows in order, so reads and writes are coalesced.
__global__ void __launch_bounds__(kPermThreads) perm_importance_gather_kernel(
    const float* __restrict__ x, int N, long row_elems, const int32_t* __restrict__ col_group, int g, int r,
    uint64_t seed, int a, int n, float* __restrict__ out) {
  __shared__ int donor[kPermRows];
  const int i0 = blockIdx.x * kPermRows;
  if (threadIdx.x < kPermRows && i0 + (int)threadIdx.x < n)
    donor[threadIdx.x] = (int)perm_index(N, seed, g, r, (uint32_t)(a + i0 + threadIdx.x));
  __syncthreads();
  const int rows = min(kPermRows, n - i0);
  for (int k = 0; k < rows; ++k) {
    const float* own = x + (long)(a + i0 + k) * row_elems;
    const float* don = x + (long)donor[k] * row_elems;
    float* dst = out + (long)(i0 + k) * row_elems;
    for (long c = threadIdx.x; c < row_elems; c += kPermThreads) dst[c] = (__ldg(col_group + c) == g ? don : own)[c];
  }
}

}  // namespace

int perm_importance_gather(cudaStream_t s, const float* x, int N, long row_elems, const int32_t* col_group, int g, int r,
                           uint64_t seed, int a, int n, float* out) {
  perm_importance_gather_kernel<<<(n + kPermRows - 1) / kPermRows, kPermThreads, 0, s>>>(x, N, row_elems, col_group, g,
                                                                                        r, seed, a, n, out);
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
