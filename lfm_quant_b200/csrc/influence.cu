// Training-window attributions (lfmq_influence_*, DESIGN.md section 5i): TracIn at the trained checkpoint, restricted to
// the output head.  The influence of training window t on output j of query q is I_j(t, q) = -s_jq (a_q . u_jt), one
// GEMM per output over vectors of length D1 = D + 1.
//
// influence_grad: per training window the one-window loss gradient G at the head output (same expressions as the
// training loss kernels, with the window's own mask counts as denominators and no row weights; masked elements give 0),
// then u_j = sum_tau G_j[tau] (a_tau; 1) in increasing tau.
// influence_query: a_q = (a_{q,T-1}; 1) and s_jq.
//
// influence_topk: the hot path.  A CTA owns 128 query rows (two consumer warpgroups of m64n128k8 tf32 wgmma), one
// output j and one slice of the pool, and walks the slice's 128-window tiles.  Operands are split 3xTF32 style while
// they are staged K-major into 128-byte-swizzled shared memory (hi = rna(v), lo = rna(v - hi)), and each k step runs
// lo*hi, hi*lo and hi*hi into one fp32 accumulator.  A score sums its k tiles in increasing order, and zero padding
// adds exact zeros, so it does not depend on the tile it lands in.  The epilogue keeps, per (row, sign), a threshold in
// shared memory: the K-th entry of the running list once it is full, else 0.  Scores of the right sign at or beyond
// it are appended to a per-(row, sign) candidate buffer, which its owner thread inserts into the running list (in
// global memory) when it could overflow in the next round.  Lists are ordered by (score, lower index first); every
// dropped score is beaten by K listed ones, so the lists are the exact top K of the slice whatever the order of
// appends.  influence_merge merges the slices' lists in slice order.
//
// total = -s_jq (a_q . sum_t u_jt): fixed blocks of pool rows summed in fp64, the blocks in order, one warp per query.
//
// lfmq_nearest_topk is the same kernel in its second mode (kNearest): the pool is b [Nt][D1], J = 1, and the score of
// pool row t is 2 (a . b_t) - |b_t|^2, with |b_t|^2 an fp64 sum in a fixed order rounded to fp32 and passed in S.  It
// keeps one list, of the largest scores whatever their sign (the nearest rows), in the sign-0 slot; its threshold is
// -inf until the list is full.  The score only shortlists: for a query near a pool row it is |a|^2 - d^2, a difference
// of large numbers, and the fp32 accumulation of the product errs by about 1e-5 of |a|^2 + |b|^2 at D1 ~ 1500, far
// more than a small d^2.  So the GEMM keeps Kc = nearest_candidates(K) = K + 16 candidates, and nearest_finish merges the
// slices, recomputes each candidate's distance exactly from the difference a - b_t in fp64, and keeps the K nearest.
#include <algorithm>
#include <atomic>

#include "kernels.h"
#include "sm90.cuh"

namespace lfmq {
namespace {

using namespace sm90;

__device__ __forceinline__ float sigmoid_g(float x) { return 1.0f / (1.0f + expf(-x)); }

// ---- features ---------------------------------------------------------------------------------------------------
constexpr int kFeatThreads = 256;

// One CTA per window b of the launch.  mode 0 point, 1 uq, 2 dense.  a: head inputs [n][Ta][D] (Ta = T, or 1 on a dense
// handle where a is the flattened window); pred / var / pre / y: [n][Ta][O].  u: [J][ldu][D1], rows from r0.
__global__ void __launch_bounds__(kFeatThreads) influence_grad_kernel(int mode, int Ta, int D, int O, int tidx, float p1,
                                                                      float p2, int huber, float delta,
                                                                      const float* __restrict__ a,
                                                                      const float* __restrict__ pred,
                                                                      const float* __restrict__ var,
                                                                      const float* __restrict__ pre,
                                                                      const float* __restrict__ y, long r0, long ldu,
                                                                      float* __restrict__ u) {
  extern __shared__ float g_s[];      // [J][Ta] gradients, then [Ta] masks
  const int b = blockIdx.x;
  const int J = mode == 1 ? 2 : 1;
  float* m_s = g_s + J * Ta;
  for (int t = threadIdx.x; t < Ta; t += blockDim.x) m_s[t] = row_mask(y + ((long)b * Ta + t) * O, O) ? 1.f : 0.f;
  __syncthreads();
  if (threadIdx.x == 0) {
    float ms_all = 0.f;
    for (int t = 0; t < Ta; ++t) ms_all += m_s[t];
    const float ms_last = m_s[Ta - 1];
    for (int t = 0; t < Ta; ++t) {
      const long e = ((long)b * Ta + t) * O + tidx;
      const float m = m_s[t];
      const bool last = t == Ta - 1;
      float g0 = 0.f, g1 = 0.f;
      if (m != 0.f && mode == 0) {            // point_loss_row with denominators {B = 1, unmasked rows of the window}
        const LossWeights lw = loss_weights(p1, p2, O, ms_all, 1.f, nullptr);
        const float d = pred[e] * m - y[e];
        float coef = lw.all;
        if (last) {
          coef += lw.last;
          coef += lw.tar;
        }
        g0 = 2.f * d * coef * m;
      } else if (m != 0.f && mode == 1) {     // uq_loss_rows with the window's counts
        const LossWeights lw = loss_weights(p1, p2, O, ms_all, ms_last, nullptr);
        const float pm = pred[e] * m, vm = var[e] * m;
        const float d = pm - y[e];
        const float diff = d * d;
        float coef = lw.all;
        if (last) {
          coef += lw.last;
          coef += lw.tar;
        }
        g0 = coef * (2.f * d / vm) * m;
        const float dv = coef * (-diff / (vm * vm) + 1.f / vm) * m;
        g1 = dv * ((softplus_f(pre[e]) > 1e-6f) ? sigmoid_g(pre[e]) : 0.f);
      } else if (m != 0.f) {                  // dense_loss_rows at B = 1
        const float g = (1.f - p1) / (1.f * (float)O) + p1 / 1.f;
        const float r = y[e] - pred[e] * m;
        const float ar = fabsf(r);
        const float df = (huber && ar > delta) ? copysignf(delta, r) : (huber ? r : 2.f * r);
        g0 = -m * g * df;
      }
      g_s[t] = g0;
      if (J == 2) g_s[Ta + t] = g1;
    }
  }
  __syncthreads();
  const int D1 = D + 1;
  for (int j = 0; j < J; ++j) {
    float* ur = u + ((long)j * ldu + r0 + b) * D1;
    for (int d = threadIdx.x; d < D1; d += blockDim.x) {
      float acc = 0.f;
      for (int t = 0; t < Ta; ++t) acc = fmaf(g_s[j * Ta + t], d < D ? a[((long)b * Ta + t) * D + d] : 1.f, acc);
      ur[d] = acc;
    }
  }
}

// One thread per element of a [n][D1]: a_out = (a[b, Ta-1, :]; 1); s [J][lds] from r0: 1, and on a uq handle
// sigmoid(pre) where the variance floor does not bind.
__global__ void influence_query_kernel(int n, int Ta, int D, int O, int tidx, int uq, const float* __restrict__ a,
                                       const float* __restrict__ pre, long r0, long lds, float* __restrict__ aout,
                                       float* __restrict__ s) {
  const int D1 = D + 1;
  const long i = (long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (long)n * D1) return;
  const long b = i / D1;
  const int d = (int)(i - b * D1);
  aout[(r0 + b) * D1 + d] = d < D ? a[(b * Ta + Ta - 1) * D + d] : 1.f;
  if (d == 0) {
    s[r0 + b] = 1.f;
    if (uq) {
      const float p = pre[(b * Ta + Ta - 1) * O + tidx];
      s[lds + r0 + b] = (softplus_f(p) > 1e-6f) ? sigmoid_g(p) : 0.f;
    }
  }
}

// ---- top-K ------------------------------------------------------------------------------------------------------
constexpr int TM = 128, TN = 128, TK = 32;
constexpr int NT = 256;
constexpr int TILE = TM * TK;
constexpr int PER_T = TILE / NT;
constexpr int CAP = 32;                        // candidates per (row, sign) between merges
constexpr int CG = 2;                          // column groups of 8 per epilogue round: <= 8 * CG appends per round
constexpr int STAGE_FLOATS = 4 * TILE;         // A hi, A lo, B hi, B lo
constexpr size_t TOPK_SMEM = (size_t)2 * STAGE_FLOATS * 4 + (size_t)TM * 2 * CAP * 8 + (size_t)TM * 2 * 3 * 4 + 1024;

__host__ __device__ inline long cdivl(long a, long b) { return (a + b - 1) / b; }

__device__ __forceinline__ int swz(int r, int k) { return r * TK + (((k >> 2) ^ (r & 7)) << 2) + (k & 3); }

// rows [r0, r0 + 128) x k [k0, k0 + 32) of a row-major [R][D1] matrix, zero outside
__device__ __forceinline__ void load_tile(float (&v)[PER_T], const float* __restrict__ P, long R, int D1, long r0,
                                          int k0, int tid) {
#pragma unroll
  for (int i = 0; i < PER_T; ++i) {
    const int k = tid & (TK - 1), r = (tid >> 5) + (NT / TK) * i;
    const long gr = r0 + r;
    const int gk = k0 + k;
    v[i] = (gr < R && gk < D1) ? __ldg(P + gr * D1 + gk) : 0.f;
  }
}

__device__ __forceinline__ void store_split(const float (&v)[PER_T], uint32_t* hi, uint32_t* lo, int tid) {
#pragma unroll
  for (int i = 0; i < PER_T; ++i) {
    const int k = tid & (TK - 1), r = (tid >> 5) + (NT / TK) * i;
    const uint32_t h = cvt_rna_tf32(v[i]);
    hi[swz(r, k)] = h;
    lo[swz(r, k)] = cvt_rna_tf32(v[i] - __uint_as_float(h));
  }
}

// a ranks before b: the larger score (pos) or the smaller (neg), ties to the lower index
__device__ __forceinline__ bool before(float as, int ai, float bs, int bi, bool neg) {
  return (neg ? as < bs : as > bs) || (as == bs && ai < bi);
}

// Inserts the n candidates into the sorted list (ls, li) of *len <= K entries; returns the new threshold.
__device__ float merge_list(float* __restrict__ ls, int* __restrict__ li, int* len, int K, const float* cs,
                            const int* ci, int n, bool neg) {
  int L = *len;
  for (int c = 0; c < n; ++c) {
    const float sc = cs[c];
    const int ix = ci[c];
    if (L == K && !before(sc, ix, ls[K - 1], li[K - 1], neg)) continue;
    int p = L < K ? L : K - 1;
    while (p > 0 && before(sc, ix, ls[p - 1], li[p - 1], neg)) {
      ls[p] = ls[p - 1];
      li[p] = li[p - 1];
      --p;
    }
    ls[p] = sc;
    li[p] = ix;
    if (L < K) ++L;
  }
  *len = L;
  return L == K ? ls[K - 1] : 0.f;
}

constexpr int kDot = 0, kNearest = 1;

// grid (query tiles, slices, J).  lists: score [J][P][Nq][2][K] and index alike, the slice's running lists.  MODE kDot:
// S [J][Nq] the s_jq; kNearest: S [Nt] the pool rows' squared norms.
template <int MODE>
__global__ void __launch_bounds__(NT, 1) influence_topk_kernel(const float* __restrict__ A, const float* __restrict__ U,
                                                               const float* __restrict__ S, int Nq, int Nt, int D1,
                                                               int K, int tiles_per_slice, float* __restrict__ lscore,
                                                               int* __restrict__ lidx) {
  extern __shared__ uint8_t smem_raw[];
  uint32_t* sm = reinterpret_cast<uint32_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
  float* cs = reinterpret_cast<float*>(sm + 2 * STAGE_FLOATS);    // [TM][2][CAP]
  int* ci = reinterpret_cast<int*>(cs + TM * 2 * CAP);             // [TM][2][CAP]
  float* thr = reinterpret_cast<float*>(ci + TM * 2 * CAP);        // [TM][2]
  int* ccnt = reinterpret_cast<int*>(thr + TM * 2);                // [TM][2]
  int* lcnt = ccnt + TM * 2;                                       // [TM][2]

  const int tid = threadIdx.x, wg = tid >> 7, wtid = tid & 127;
  const int j = blockIdx.z, P = gridDim.y, p = blockIdx.y;
  const long q0 = (long)blockIdx.x * TM;
  const float* Uj = U + (long)j * Nt * D1;
  const long ntiles = cdivl(Nt, TN);
  const long tile0 = (long)p * tiles_per_slice;
  const long tile1 = min(ntiles, tile0 + tiles_per_slice);
  const int nk = (int)cdivl(D1, TK);
  const long iters = (tile1 - tile0) * nk;

  // the (row, sign) this thread owns: row = 64 wg + wtid / 2, sign = wtid & 1
  const int orow = 64 * wg + (wtid >> 1), osgn = wtid & 1;
  const long oq = q0 + orow;
  float* my_ls = lscore + ((((long)j * P + p) * Nq + oq) * 2 + osgn) * K;
  int* my_li = lidx + ((((long)j * P + p) * Nq + oq) * 2 + osgn) * K;
  thr[orow * 2 + osgn] = MODE == kNearest ? -INFINITY : 0.f;
  ccnt[orow * 2 + osgn] = 0;
  lcnt[orow * 2 + osgn] = 0;

  const int w = (tid >> 5) & 3, l = tid & 31;
  const int rl0 = 64 * wg + 16 * w + (l >> 2);      // rows rl0 and rl0 + 8 of the CTA tile
  float srow[2] = {0.f, 0.f};
  if constexpr (MODE == kDot)
    for (int h = 0; h < 2; ++h) {
      const long q = q0 + rl0 + 8 * h;
      srow[h] = q < Nq ? S[(long)j * Nq + q] : 0.f;
    }

  float acc[64];
  float va[PER_T], vb[PER_T];
  if (iters > 0) {
    load_tile(va, A, Nq, D1, q0, 0, tid);
    load_tile(vb, Uj, Nt, D1, tile0 * TN, 0, tid);
    store_split(va, sm, sm + TILE, tid);
    store_split(vb, sm + 2 * TILE, sm + 3 * TILE, tid);
  }
  fence_proxy_async_smem();
  __syncthreads();

  for (long it = 0; it < iters; ++it) {
    const int kt = (int)(it % nk);
    const long nt = tile0 + it / nk;
    const int st = (int)(it & 1);
    const bool more = it + 1 < iters;
    if (kt == 0) {
#pragma unroll
      for (int i = 0; i < 64; ++i) acc[i] = 0.f;
    }
    if (more) {
      const int kn = (int)((it + 1) % nk);
      const long tn = tile0 + (it + 1) / nk;
      load_tile(va, A, Nq, D1, q0, kn * TK, tid);
      load_tile(vb, Uj, Nt, D1, tn * TN, kn * TK, tid);
    }
    uint32_t* stage = sm + st * STAGE_FLOATS;
    const uint32_t a_hi = smem_u32(stage) + wg * 64 * TK * 4, a_lo = smem_u32(stage + TILE) + wg * 64 * TK * 4;
    const uint32_t b_hi = smem_u32(stage + 2 * TILE), b_lo = smem_u32(stage + 3 * TILE);
    wgmma_fence();
#pragma unroll
    for (int kk = 0; kk < TK / 8; ++kk) {
      const uint64_t dah = make_smem_desc(a_hi + kk * 32, 0, 1024, LAYOUT_SW128);
      const uint64_t dal = make_smem_desc(a_lo + kk * 32, 0, 1024, LAYOUT_SW128);
      const uint64_t dbh = make_smem_desc(b_hi + kk * 32, 0, 1024, LAYOUT_SW128);
      const uint64_t dbl = make_smem_desc(b_lo + kk * 32, 0, 1024, LAYOUT_SW128);
      wgmma_m64n128k8_tf32(acc, dal, dbh, 1);
      wgmma_m64n128k8_tf32(acc, dah, dbl, 1);
      wgmma_m64n128k8_tf32(acc, dah, dbh, 1);
    }
    wgmma_commit();
    if (more) {
      uint32_t* nx = sm + (st ^ 1) * STAGE_FLOATS;
      store_split(va, nx, nx + TILE, tid);
      store_split(vb, nx + 2 * TILE, nx + 3 * TILE, tid);
    }
    wgmma_wait<0>();
    fence_regs(acc);

    if (kt == nk - 1) {      // epilogue of tile nt: this warpgroup's 64 rows, in rounds of CG column groups
      const long n0 = nt * TN;
#pragma unroll
      for (int r = 0; r < 16 / CG; ++r) {
#pragma unroll
        for (int i = r * CG * 4; i < (r + 1) * CG * 4; ++i) {
          const int h = (i >> 1) & 1;
          const int row = rl0 + 8 * h;
          const long t = n0 + 8 * (i >> 2) + 2 * (l & 3) + (i & 1);
          if constexpr (MODE == kNearest) {
            if (t < Nt) {
              const float sc = 2.f * acc[i] - __ldg(S + t);
              if (sc >= thr[row * 2]) {
                const int slot = atomicAdd(&ccnt[row * 2], 1);
                cs[(row * 2) * CAP + slot] = sc;
                ci[(row * 2) * CAP + slot] = (int)t;
              }
            }
            continue;
          }
          const float sc = -(srow[h] * acc[i]);
          if (t < Nt) {
            if (sc > 0.f && sc >= thr[row * 2]) {
              const int slot = atomicAdd(&ccnt[row * 2], 1);
              cs[(row * 2) * CAP + slot] = sc;
              ci[(row * 2) * CAP + slot] = (int)t;
            } else if (sc < 0.f && sc <= thr[row * 2 + 1]) {
              const int slot = atomicAdd(&ccnt[row * 2 + 1], 1);
              cs[(row * 2 + 1) * CAP + slot] = sc;
              ci[(row * 2 + 1) * CAP + slot] = (int)t;
            }
          }
        }
        named_bar_sync(1 + wg, 128);
        const int o = orow * 2 + osgn;
        const bool flush = (r == 16 / CG - 1) && (it + 1 == iters);
        if (ccnt[o] > CAP - 8 * CG || (flush && ccnt[o] > 0)) {
          int len = lcnt[o];
          if (oq < Nq) thr[o] = merge_list(my_ls, my_li, &len, K, cs + o * CAP, ci + o * CAP, ccnt[o], osgn == 1);
          if (MODE == kNearest && len < K) thr[o] = -INFINITY;
          lcnt[o] = len;
          ccnt[o] = 0;
        }
        named_bar_sync(1 + wg, 128);
      }
    }
    fence_proxy_async_smem();
    __syncthreads();
  }
  if (oq < Nq)
    for (int k = lcnt[orow * 2 + osgn]; k < K; ++k) {
      my_ls[k] = 0.f;
      my_li[k] = -1;
    }
}

// One thread per (j, q, sign): the P slice lists inserted, in slice order, into the output list, then padded.
__global__ void influence_merge_kernel(int Nq, int J, int P, int K, const float* __restrict__ lscore,
                                       const int* __restrict__ lidx, int* __restrict__ pos_idx,
                                       float* __restrict__ pos_score, int* __restrict__ neg_idx,
                                       float* __restrict__ neg_score) {
  const long i = (long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (long)J * Nq * 2) return;
  const int sgn = (int)(i & 1);
  const long q = (i >> 1) % Nq;
  const int j = (int)((i >> 1) / Nq);
  int* oi = (sgn ? neg_idx : pos_idx) + (q * J + j) * K;
  float* os = (sgn ? neg_score : pos_score) + (q * J + j) * K;
  int len = 0;
  for (int p = 0; p < P; ++p) {
    const long e = ((((long)j * P + p) * Nq + q) * 2 + sgn) * K;
    int n = 0;
    while (n < K && lidx[e + n] >= 0) ++n;
    merge_list(os, oi, &len, K, lscore + e, lidx + e, n, sgn == 1);
  }
  for (int k = len; k < K; ++k) {
    oi[k] = -1;
    os[k] = 0.f;
  }
}

constexpr int kFinishWarps = 4;

// One warp per query.  Lane 0 merges the P slices' sign-0 lists of Kc candidates in slice order (by the GEMM's score);
// the warp then forms every candidate's exact squared distance |a - b_t|^2 from the difference in fp64 (lanes strided
// over the columns, then a fixed butterfly), and lane 0 sorts the candidates by (distance, index) and writes the first
// K: idx and d2, padded with -1 / +inf past the pool, and mean = their values summed in rank order in fp64 over their
// count.
__global__ void __launch_bounds__(32 * kFinishWarps) nearest_finish_kernel(int Nq, int P, int Kc, int K,
                                                                           const float* __restrict__ lscore,
                                                                           const int* __restrict__ lidx,
                                                                           const float* __restrict__ a,
                                                                           const float* __restrict__ b, int D1,
                                                                           const float* __restrict__ value,
                                                                           int32_t* __restrict__ idx,
                                                                           float* __restrict__ d2,
                                                                           float* __restrict__ mean) {
  __shared__ float cs[kFinishWarps][LFMQ_NEAREST_MAX_CAND];
  __shared__ int ci[kFinishWarps][LFMQ_NEAREST_MAX_CAND];
  __shared__ double cd[kFinishWarps][LFMQ_NEAREST_MAX_CAND];
  const int w = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const long q = (long)blockIdx.x * kFinishWarps + w;
  if (q >= Nq) return;                       // the whole warp
  int len = 0;
  if (lane == 0)
    for (int p = 0; p < P; ++p) {
      const long e = (((long)p * Nq + q) * 2) * Kc;
      int n = 0;
      while (n < Kc && lidx[e + n] >= 0) ++n;
      merge_list(cs[w], ci[w], &len, Kc, lscore + e, lidx + e, n, false);
    }
  len = __shfl_sync(0xffffffffu, len, 0);
  __syncwarp();
  const float* aq = a + q * D1;
  for (int c = 0; c < len; ++c) {
    const float* bt = b + (long)ci[w][c] * D1;
    double acc = 0.0;
    for (int d = lane; d < D1; d += 32) {
      const double v = (double)aq[d] - (double)bt[d];
      acc += v * v;
    }
    acc = warp_sum(acc);
    if (lane == 0) cd[w][c] = acc;
  }
  __syncwarp();
  if (lane != 0) return;
  for (int c = 1; c < len; ++c) {            // insertion sort by (distance, lower index)
    const double dv = cd[w][c];
    const int iv = ci[w][c];
    int p = c;
    while (p > 0 && (cd[w][p - 1] > dv || (cd[w][p - 1] == dv && ci[w][p - 1] > iv))) {
      cd[w][p] = cd[w][p - 1];
      ci[w][p] = ci[w][p - 1];
      --p;
    }
    cd[w][p] = dv;
    ci[w][p] = iv;
  }
  const int n = len < K ? len : K;
  double acc = 0.0;
  for (int k = 0; k < K; ++k) {
    if (k < n) {
      idx[q * K + k] = ci[w][k];
      d2[q * K + k] = (float)cd[w][k];
      if (value) acc += (double)value[ci[w][k]];
    } else {
      idx[q * K + k] = -1;
      d2[q * K + k] = INFINITY;
    }
  }
  if (value) mean[q] = (float)(acc / n);
}

// One warp per row of p [R][D1]: the squared norm, lanes strided over the columns in fp64, then a fixed butterfly,
// rounded to fp32.
__global__ void nearest_norm_kernel(const float* __restrict__ p, int R, int D1, float* __restrict__ nf) {
  const long r = ((long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  if (r >= R) return;
  double acc = 0.0;
  for (int d = threadIdx.x & 31; d < D1; d += 32) {
    const double v = (double)p[r * D1 + d];
    acc += v * v;
  }
  acc = warp_sum(acc);
  if ((threadIdx.x & 31) == 0) nf[r] = (float)acc;
}

template <int MODE>
int configure_topk() {
  static std::atomic<uint64_t> configured{0};
  int dev = 0;
  LFMQ_CUDA_CHECK(cudaGetDevice(&dev));
  const uint64_t bit = 1ull << (dev & 63);
  if (!(configured.load() & bit)) {
    LFMQ_CUDA_CHECK(cudaFuncSetAttribute(influence_topk_kernel<MODE>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                         (int)TOPK_SMEM));
    configured.fetch_or(bit);
  }
  return 0;
}

constexpr int kSumRows = 2048;     // pool rows per partial sum of sum_t u_t

// grid (ceil(D1 / 128), ceil(Nt / kSumRows), J): part[j][blk][d] = sum of rows [blk * kSumRows, ...) in increasing t
__global__ void influence_usum_kernel(const float* __restrict__ U, int Nt, int D1, double* __restrict__ part) {
  const int d = blockIdx.x * blockDim.x + threadIdx.x;
  if (d >= D1) return;
  const int j = blockIdx.z, blk = blockIdx.y;
  const float* Uj = U + (long)j * Nt * D1;
  const long t1 = min((long)Nt, (long)(blk + 1) * kSumRows);
  double acc = 0.0;
  for (long t = (long)blk * kSumRows; t < t1; ++t) acc += (double)Uj[t * D1 + d];
  part[((long)j * gridDim.y + blk) * D1 + d] = acc;
}

// usum[j][d] = the nb partials summed in block order
__global__ void influence_usum_final_kernel(const double* __restrict__ part, int nb, int D1, int J,
                                            double* __restrict__ usum) {
  const long i = (long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (long)J * D1) return;
  const long j = i / D1, d = i - j * D1;
  double acc = 0.0;
  for (int b = 0; b < nb; ++b) acc += part[(j * nb + b) * D1 + d];
  usum[i] = acc;
}

// one warp per (q, j): total[q][j] = -s_jq (a_q . usum_j), fp64, lanes then a fixed butterfly
__global__ void influence_total_kernel(const float* __restrict__ A, const float* __restrict__ S,
                                       const double* __restrict__ usum, int Nq, int D1, int J,
                                       float* __restrict__ total) {
  const long wid = ((long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  if (wid >= (long)Nq * J) return;
  const long q = wid / J;
  const int j = (int)(wid - q * J);
  double acc = 0.0;
  for (int d = threadIdx.x & 31; d < D1; d += 32) acc += (double)A[q * D1 + d] * usum[(long)j * D1 + d];
  acc = warp_sum(acc);
  if ((threadIdx.x & 31) == 0) total[q * J + j] = (float)(-(double)S[(long)j * Nq + q] * acc);
}

}  // namespace

int influence_grad(cudaStream_t s, int n, int mode, int Ta, int D, int O, int tidx, float p1, float p2, int huber,
                   float delta, const float* a, const float* pred, const float* var, const float* pre, const float* y,
                   long r0, long ldu, float* u) {
  if (n <= 0) return 0;
  const size_t smem = (size_t)((mode == 1 ? 2 : 1) + 1) * Ta * sizeof(float);
  influence_grad_kernel<<<n, kFeatThreads, smem, s>>>(mode, Ta, D, O, tidx, p1, p2, huber, delta, a, pred, var, pre, y,
                                                      r0, ldu, u);
  LFMQ_LAUNCH_CHECK();
  return 0;
}

int influence_query(cudaStream_t s, int n, int Ta, int D, int O, int tidx, int uq, const float* a, const float* pre,
                    long r0, long lds, float* aout, float* sout) {
  if (n <= 0) return 0;
  const long total = (long)n * (D + 1);
  influence_query_kernel<<<(int)cdivl(total, 256), 256, 0, s>>>(n, Ta, D, O, tidx, uq, a, pre, r0, lds, aout, sout);
  LFMQ_LAUNCH_CHECK();
  return 0;
}

InfluencePlan influence_plan(int Nq, int Nt, int D1, int J, int K) {
  InfluencePlan pl;
  const long qt = cdivl(Nq, TM), ntiles = cdivl(Nt, TN);
  // about two CTAs per SM of an H100 (132 SMs) in all, at most 64 slices, at least one tile each
  long P = cdivl(264, qt * J);
  P = std::max(1L, std::min(P, std::min(ntiles, 64L)));
  pl.tiles_per_slice = (int)cdivl(ntiles, P);
  pl.P = (int)cdivl(ntiles, pl.tiles_per_slice);
  pl.n_sum = (int)cdivl(Nt, kSumRows);
  pl.list_elems = (size_t)J * pl.P * Nq * 2 * K;
  pl.part_elems = (size_t)J * pl.n_sum * D1;
  pl.usum_elems = (size_t)J * D1;
  return pl;
}

int influence_topk(cudaStream_t s, const InfluencePlan& pl, const float* a, const float* u, const float* sc, int Nq,
                   int Nt, int D1, int J, int K, float* lscore, int* lidx, double* part, double* usum, int* pos_idx,
                   float* pos_score, int* neg_idx, float* neg_score, float* total) {
  if (int e = configure_topk<kDot>()) return e;
  const dim3 grid((unsigned)cdivl(Nq, TM), (unsigned)pl.P, (unsigned)J);
  influence_topk_kernel<kDot><<<grid, NT, TOPK_SMEM, s>>>(a, u, sc, Nq, Nt, D1, K, pl.tiles_per_slice, lscore, lidx);
  LFMQ_LAUNCH_CHECK();
  const long nm = (long)J * Nq * 2;
  influence_merge_kernel<<<(int)cdivl(nm, 128), 128, 0, s>>>(Nq, J, pl.P, K, lscore, lidx, pos_idx, pos_score, neg_idx,
                                                            neg_score);
  LFMQ_LAUNCH_CHECK();
  influence_usum_kernel<<<dim3((unsigned)cdivl(D1, 128), (unsigned)pl.n_sum, (unsigned)J), 128, 0, s>>>(u, Nt, D1,
                                                                                                        part);
  LFMQ_LAUNCH_CHECK();
  influence_usum_final_kernel<<<(int)cdivl((long)J * D1, 128), 128, 0, s>>>(part, pl.n_sum, D1, J, usum);
  LFMQ_LAUNCH_CHECK();
  influence_total_kernel<<<(int)cdivl((long)Nq * J * 32, 256), 256, 0, s>>>(a, sc, usum, Nq, D1, J, total);
  LFMQ_LAUNCH_CHECK();
  return 0;
}

int nearest_norms(cudaStream_t s, const float* p, int R, int D1, float* nf) {
  nearest_norm_kernel<<<(int)cdivl((long)R * 32, 256), 256, 0, s>>>(p, R, D1, nf);
  LFMQ_LAUNCH_CHECK();
  return 0;
}

int nearest_topk(cudaStream_t s, const InfluencePlan& pl, const float* a, const float* b, const float* bn,
                 const float* value, int Nq, int Nt, int D1, int K, float* lscore, int* lidx, int32_t* idx, float* d2,
                 float* mean) {
  const int Kc = nearest_candidates(K);
  if (int e = configure_topk<kNearest>()) return e;
  const dim3 grid((unsigned)cdivl(Nq, TM), (unsigned)pl.P, 1u);
  influence_topk_kernel<kNearest><<<grid, NT, TOPK_SMEM, s>>>(a, b, bn, Nq, Nt, D1, Kc, pl.tiles_per_slice, lscore,
                                                              lidx);
  LFMQ_LAUNCH_CHECK();
  nearest_finish_kernel<<<(int)cdivl(Nq, kFinishWarps), 32 * kFinishWarps, 0, s>>>(Nq, pl.P, Kc, K, lscore, lidx, a, b,
                                                                                 D1, value, idx, d2, mean);
  LFMQ_LAUNCH_CHECK();
  return 0;
}

}  // namespace lfmq
