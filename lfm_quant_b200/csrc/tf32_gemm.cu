// The GEMMs of a LFMQ_PREC_TF32 handle: the fp32 path's strided products on sm_90a wgmma with tf32 operands and fp32
// accumulation.  Same arguments and split-K rule as sgemm (kernels_simt.cu), so forward_fp32 / backward_fp32 call
// either through one dispatch.
//
// tf32 wgmma has no transpose immediates: both shared-memory operands must be K-major.  The step's operands come in
// all four layouts (W and U are [K][N], the weight gradients read both operands MN-major), so every tile is staged
// through registers: each thread loads its elements with coalesced loads along whichever axis is contiguous in memory,
// rounds them with cvt.rna.tf32.f32 and stores them K-major into a 128-byte-swizzled shared-memory tile.  The rounding
// is therefore explicit (nearest, ties away from zero) wherever an operand enters a product, whatever wgmma does with
// the low mantissa bits.  Loads are bounds-checked (zero fill), so M, N and K are arbitrary and no address or stride
// needs alignment.  The next k tile's loads are in flight while the current tile's wgmma runs (two shared stages).
//
// Determinism: an output element sums its k tiles in increasing order, and inside a tile the wgmma's own order; none of
// it depends on the element's row, on M or on the launch.  Split-K (only when the caller passes scratch: the weight
// gradients, K = B*T) writes partials that splitk_reduce sums in split order.  No atomics, no cross-CTA waits.
#include "kernels.h"
#include "sm90.cuh"

namespace lfmq {
namespace {

using namespace sm90;

constexpr int TM = 128, TN = 128, TK = 32;   // two consumer warpgroups of m64n128, k tiles of 32 (one 128-byte row)
constexpr int NT = 256;
constexpr int TILE = TM * TK;                 // floats of one operand tile (TM == TN)
constexpr int PER_T = TILE / NT;              // elements each thread stages per operand tile
constexpr int SMEM_BYTES = 2 * 2 * TILE * 4 + 1024;

__host__ __device__ inline int cdiv(long a, long b) { return (int)((a + b - 1) / b); }

// element (r, k) of a K-major tile with the 128-byte swizzle: row r is one 128-byte line of 32 k values, whose eight
// 16-byte chunks are permuted by r % 8 (the layout a SWIZZLE_128B descriptor reads)
__device__ __forceinline__ int swz(int r, int k) { return r * TK + (((k >> 2) ^ (r & 7)) << 2) + (k & 3); }

// this thread's (row, k) of element i of a tile: consecutive threads walk the axis that is contiguous in memory
template <bool MN_CONTIG>
__device__ __forceinline__ void tile_pos(int tid, int i, int& r, int& k) {
  if (MN_CONTIG) {
    r = tid & (TM - 1);
    k = (tid >> 7) + (NT / TM) * i;
  } else {
    k = tid & (TK - 1);
    r = (tid >> 5) + (NT / TK) * i;
  }
}

// P(r, k) = P[r * s_r + k * s_k] for rows [r0, r0 + 128) and k in [k0, k0 + 32), zero outside [0, R) x [.., kend)
template <bool MN_CONTIG>
__device__ __forceinline__ void load_tile(float (&v)[PER_T], const float* __restrict__ P, long s_r, long s_k, int r0,
                                          int R, int k0, int kend, int tid) {
#pragma unroll
  for (int i = 0; i < PER_T; ++i) {
    int r, k;
    tile_pos<MN_CONTIG>(tid, i, r, k);
    const int gr = r0 + r, gk = k0 + k;
    v[i] = (gr < R && gk < kend) ? __ldg(P + (long)gr * s_r + (long)gk * s_k) : 0.f;
  }
}

template <bool MN_CONTIG>
__device__ __forceinline__ void store_tile(const float (&v)[PER_T], uint32_t* S, int tid) {
#pragma unroll
  for (int i = 0; i < PER_T; ++i) {
    int r, k;
    tile_pos<MN_CONTIG>(tid, i, r, k);
    S[swz(r, k)] = cvt_rna_tf32(v[i]);
  }
}

// C[M,N] = A*B + beta*C (or, with `partial`, split z's product into partial[z][M][N]); A(m,k) = A[m*sAm + k*sAk],
// B(k,n) = B[k*sBk + n*sBn]; blockIdx.z covers k in [z * kchunk, min(K, (z + 1) * kchunk)).
template <bool A_M_CONTIG, bool B_N_CONTIG>
__global__ void __launch_bounds__(NT) tf32_gemm_kernel(int M, int N, int K, const float* __restrict__ A, long sAm,
                                                       long sAk, const float* __restrict__ B, long sBk, long sBn,
                                                       float* __restrict__ C, long ldc, float beta, int kchunk,
                                                       float* __restrict__ partial) {
  extern __shared__ uint8_t smem_raw[];
  uint32_t* sm = reinterpret_cast<uint32_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
  const int tid = threadIdx.x, wg = tid >> 7;
  const int m0 = blockIdx.y * TM, n0 = blockIdx.x * TN;
  const int kbeg = blockIdx.z * kchunk;
  const int kend = min(K, kbeg + kchunk);
  const int nk = max(1, cdiv(kend - kbeg, TK));

  float acc[64];
#pragma unroll
  for (int i = 0; i < 64; ++i) acc[i] = 0.f;
  float va[PER_T], vb[PER_T];
  load_tile<A_M_CONTIG>(va, A, sAm, sAk, m0, M, kbeg, kend, tid);
  load_tile<B_N_CONTIG>(vb, B, sBn, sBk, n0, N, kbeg, kend, tid);
  store_tile<A_M_CONTIG>(va, sm, tid);
  store_tile<B_N_CONTIG>(vb, sm + TILE, tid);
  fence_proxy_async_smem();
  __syncthreads();

  for (int kt = 0; kt < nk; ++kt) {
    const int st = kt & 1;
    const bool more = kt + 1 < nk;
    if (more) {      // the next tile's global loads overlap this tile's MMAs
      const int k0 = kbeg + (kt + 1) * TK;
      load_tile<A_M_CONTIG>(va, A, sAm, sAk, m0, M, k0, kend, tid);
      load_tile<B_N_CONTIG>(vb, B, sBn, sBk, n0, N, k0, kend, tid);
    }
    const uint32_t a_base = smem_u32(sm + st * 2 * TILE) + wg * 64 * TK * 4;
    const uint32_t b_base = smem_u32(sm + st * 2 * TILE + TILE);
    wgmma_fence();
#pragma unroll
    for (int kk = 0; kk < TK / 8; ++kk) {       // k = 8 per wgmma: 32 bytes along each 128-byte row
      const uint64_t da = make_smem_desc(a_base + kk * 32, 0, 1024, LAYOUT_SW128);
      const uint64_t db = make_smem_desc(b_base + kk * 32, 0, 1024, LAYOUT_SW128);
      wgmma_m64n128k8_tf32(acc, da, db, 1);
    }
    wgmma_commit();
    if (more) {      // the other stage was last read by the previous tile's MMAs, complete before the last barrier
      uint32_t* nx = sm + (st ^ 1) * 2 * TILE;
      store_tile<A_M_CONTIG>(va, nx, tid);
      store_tile<B_N_CONTIG>(vb, nx + TILE, tid);
    }
    wgmma_wait<0>();
    fence_regs(acc);
    fence_proxy_async_smem();
    __syncthreads();
  }

  // accumulator fragment (sm90.cuh): row = 16 w + l / 4 + 8 ((i >> 1) & 1), col = 8 (i >> 2) + 2 (l & 3) + (i & 1)
  const int w = (tid >> 5) & 3, l = tid & 31;
#pragma unroll
  for (int i = 0; i < 64; ++i) {
    const int gm = m0 + wg * 64 + 16 * w + (l >> 2) + 8 * ((i >> 1) & 1);
    const int gn = n0 + 8 * (i >> 2) + 2 * (l & 3) + (i & 1);
    if (gm >= M || gn >= N) continue;
    if (partial) {
      partial[((long)blockIdx.z * M + gm) * N + gn] = acc[i];
    } else {
      float* c = C + (long)gm * ldc + gn;
      *c = (beta == 0.f) ? acc[i] : fmaf(beta, *c, acc[i]);
    }
  }
}

template <bool AM, bool BN>
int launch(dim3 grid, cudaStream_t s, int M, int N, int K, const float* A, long sAm, long sAk, const float* B, long sBk,
           long sBn, float* C, long ldc, float beta, int kchunk, float* partial) {
  static std::atomic<uint64_t> configured{0};      // one bit per device (ensembles run members on several GPUs)
  int dev = 0;
  LFMQ_CUDA_CHECK(cudaGetDevice(&dev));
  const uint64_t bit = 1ull << (dev & 63);
  if (!(configured.load() & bit)) {
    LFMQ_CUDA_CHECK(cudaFuncSetAttribute(tf32_gemm_kernel<AM, BN>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                         SMEM_BYTES));
    configured.fetch_or(bit);
  }
  tf32_gemm_kernel<AM, BN><<<grid, NT, SMEM_BYTES, s>>>(M, N, K, A, sAm, sAk, B, sBk, sBn, C, ldc, beta, kchunk,
                                                         partial);
  LFMQ_LAUNCH_CHECK();
  return 0;
}

}  // namespace

int tf32_gemm(cudaStream_t s, int M, int N, int K, const float* A, long sAm, long sAk, const float* B, long sBk,
              long sBn, float* C, long ldc, float beta, float* scratch, size_t scratch_elems) {
  if (M <= 0 || N <= 0) return 0;
  // split-K only with scratch (the weight gradients); the split count depends on the shape alone
  const int tiles = cdiv(M, TM) * cdiv(N, TN);
  int S = 1;
  if (K >= 2048 && tiles < 264 && scratch) {
    S = std::min(cdiv(K, 1024), std::max(1, 528 / tiles));
    while (S > 1 && (size_t)S * M * N > scratch_elems) --S;
  }
  int kchunk = cdiv(cdiv(K, S), TK) * TK;
  if (kchunk <= 0) kchunk = TK;
  S = std::max(1, cdiv(K, kchunk));
  const dim3 grid(cdiv(N, TN), cdiv(M, TM), S);
  float* partial = (S > 1) ? scratch : nullptr;
  const bool am = (sAm == 1), bn = (sBn == 1);
  auto* run = am ? (bn ? launch<true, true> : launch<true, false>) : (bn ? launch<false, true> : launch<false, false>);
  const int rc = run(grid, s, M, N, K, A, sAm, sAk, B, sBk, sBn, C, ldc, beta, kchunk, partial);
  if (rc != 0 || S == 1) return rc;
  return splitk_reduce(s, M, N, S, partial, C, ldc, beta);
}

}  // namespace lfmq
