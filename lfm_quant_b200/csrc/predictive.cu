// Predictive distributions of Monte-Carlo dropout samples (lfmq_chain_forward_uq_dist): the gather of every sample's
// (pred, var) at [T-1, target_idx], and one pass that treats each window's samples as the Gaussian mixture
// F(q) = (1/M) sum_s Phi((q - mu_s) / sigma_s) and writes its quantiles and the proper scores of the target.
// DESIGN.md section 5g.
#include "../../include/lfmq.h"
#include "kernels.h"

namespace lfmq {

namespace {

constexpr int kGatherThreads = 256;
constexpr int kDistWarps = 8;                 // (window, stage) problems per CTA, one warp each
constexpr int kQuantileIters = 64;            // safeguarded Newton: each step at least bisects when Newton stalls
// stop at |F(q) - tau| <= kQuantileRtol min(tau, 1 - tau): above the <= 4.8e-7 relative error of the fp32 erfcf terms,
// and q is then within kQuantileRtol min(tau, 1 - tau) / f(q): for one Gaussian at most 1.25e-6 sd, and 1e-6 sd / |z|
// in its tails
constexpr double kQuantileRtol = 1e-6;
constexpr float kInvSqrt2 = 0.70710678118654752f;
constexpr float kInvSqrt2Pi = 0.39894228040143268f;
constexpr double kLogSqrt2Pi = 0.91893853320467274;
constexpr double kInvSqrtPi = 0.56418958354775629;

template <typename P>
__device__ __forceinline__ P stage_ptr(const P* p, int st) {
  P r = p[0];
#pragma unroll
  for (int j = 1; j < LFMQ_MAX_STAGES; ++j)   // selects, not a dynamic index into the parameter array
    if (j == st) r = p[j];
  return r;
}

// Launch row j of tiled rows [r0, r0 + n) is sample s = (r0 + j) / B of window b = (r0 + j) mod B: its (pred, var) at
// element `off` of the row go to mu[b * samples + s] and v[b * samples + s] of every stage.
__global__ void __launch_bounds__(kGatherThreads) dist_gather_kernel(int B, int TO, long off, int64_t r0, int n,
                                                                     int samples, ChainPtrs pred, ChainPtrs var,
                                                                     ChainPtrs mu, ChainPtrs v) {
  const int j = blockIdx.x * kGatherThreads + threadIdx.x;
  if (j >= n) return;
  const int st = blockIdx.y;
  const int64_t r = r0 + j;
  const long o = (long)(r % B) * samples + (long)(r / B);
  const long src = (long)j * TO + off;
  stage_ptr(mu.p, st)[o] = stage_ptr(pred.p, st)[src];
  stage_ptr(v.p, st)[o] = stage_ptr(var.p, st)[src];
}

// The fixed-order warp sum: lane 0 adds the halves in a tree, then every lane reads lane 0's total.
__device__ __forceinline__ double warp_sum(double x) {
#pragma unroll
  for (int d = 16; d > 0; d >>= 1) x += __shfl_down_sync(0xffffffffu, x, d);
  return __shfl_sync(0xffffffffu, x, 0);
}

__device__ __forceinline__ float warp_max(float x) {
#pragma unroll
  for (int d = 16; d > 0; d >>= 1) x = fmaxf(x, __shfl_xor_sync(0xffffffffu, x, d));
  return x;
}

__device__ __forceinline__ float warp_min(float x) {
#pragma unroll
  for (int d = 16; d > 0; d >>= 1) x = fminf(x, __shfl_xor_sync(0xffffffffu, x, d));
  return x;
}

// A(m, s^2) = E|Z| for Z ~ N(m, s^2) = 2 s phi(m / s) + m (2 Phi(m / s) - 1), with 2 Phi(z) - 1 = erf(z / sqrt 2)
__device__ __forceinline__ float abs_moment(float m, float var) {
  const float inv = rsqrtf(var), z = m * inv;
  return 2.f * (var * inv) * kInvSqrt2Pi * __expf(-0.5f * z * z) + m * erff(z * kInvSqrt2);
}

// The mixture's mass below q (upper = false: F(q)) or above it (upper = true: 1 - F(q)) and its density f(q), every
// lane holding both: lane k evaluates components k, k + 32, ..  Each component's mass beyond |z|, Phi(-|z|) =
// erfc(|z| / sqrt 2) / 2, is accurate relative to itself; the other side is 1 minus it in fp64.  So both tails keep
// their relative accuracy: forming 1 - F from F would leave nothing of a 1e-4 upper tail below fp32's spacing at 1.
__device__ __forceinline__ void mixture_tail_pdf(const float* mu, const float* v, int M, double inv_m, float q,
                                                 bool upper, double* P, double* f) {
  double c = 0.0, d = 0.0;
  for (int s = threadIdx.x & 31; s < M; s += 32) {
    const float inv = rsqrtf(v[s]);
    const float z = (q - mu[s]) * inv;
    const double t = (double)(0.5f * erfcf(fabsf(z) * kInvSqrt2));
    c += ((z < 0.f) != upper) ? t : 1.0 - t;
    d += (double)(kInvSqrt2Pi * __expf(-0.5f * z * z) * inv);
  }
  *P = warp_sum(c) * inv_m;
  *f = warp_sum(d) * inv_m;
}

// log(sigma phi((y - mu) / sigma)) + log sqrt(2 pi) = -(y - mu)^2 / (2 v) - log(v) / 2, in fp64: the log score's terms
// reach -1e4 for a target far from every component, where fp32 would lose its last digits
__device__ __forceinline__ double log_kernel(float y, float mu, float v) {
  const double d = (double)y - mu, vd = v;
  const float i = rsqrtf(v);
  double r = (double)(i * i);                 // 1 / v to fp32, then two Newton steps to fp64
  r = r * (2.0 - vd * r);
  r = r * (2.0 - vd * r);
  return -0.5 * (d * d * r + log(vd));
}

struct DistParams {
  ChainCPtrs mu, v, y;          // y.p[st] nullable: no scores
  ChainPtrs q, scores;
  float levels[LFMQ_DIST_MAX_LEVELS];
  int B, M, Q;
  double inv_m;                 // 1 / M
  long y_stride, y_off;         // the target of window b: y.p[st][b * y_stride + y_off]
};

// One warp per (window, stage).  Every lane evaluates its components in fp32 and keeps its partial sums in fp64; the
// warp adds the lanes in a fixed tree (warp_sum), so a window's outputs depend on nothing but its own samples.
__global__ void __launch_bounds__(kDistWarps * 32) dist_kernel(DistParams p) {
  const int b = blockIdx.x * kDistWarps + (threadIdx.x >> 5);
  if (b >= p.B) return;
  const int st = blockIdx.y, lane = threadIdx.x & 31, M = p.M;
  const double inv_m = p.inv_m;
  const float* mu = stage_ptr(p.mu.p, st) + (long)b * M;
  const float* v = stage_ptr(p.v.p, st) + (long)b * M;

  float min_sd = INFINITY;
  for (int s = lane; s < M; s += 32) min_sd = fminf(min_sd, v[s] * rsqrtf(v[s]));
  min_sd = warp_min(min_sd);
  float* qout = stage_ptr(p.q.p, st) + (long)b * p.Q;
  for (int k = 0; k < p.Q; ++k) {
    // the root lies between the smallest and the largest component quantile: F is below tau at the one and above it
    // at the other
    const float tau = p.levels[k], zt = normcdfinvf(tau);
    float lo = INFINITY, hi = -INFINITY;
    for (int s = lane; s < M; s += 32) {
      const float qs = fmaf(v[s] * rsqrtf(v[s]), zt, mu[s]);
      lo = fminf(lo, qs);
      hi = fmaxf(hi, qs);
    }
    lo = warp_min(lo);
    hi = warp_max(hi);
    // Above the median solve 1 - F(q) = 1 - tau: g = F - tau is formed from the smaller tail, and the stop is relative
    // to it, so a level of 1e-4 or 0.9999 is met as closely, relative to its tail, as one of 0.5
    const bool upper = tau > 0.5f;
    const double t = upper ? 1.0 - (double)tau : (double)tau;
    float q = 0.5f * (lo + hi), dx = hi - lo;
    for (int it = 0; it < kQuantileIters && hi - lo > 1e-6f * min_sd; ++it) {
      double P, f;
      mixture_tail_pdf(mu, v, M, inv_m, q, upper, &P, &f);
      const double g = upper ? t - P : P - t;
      if (fabs(g) <= kQuantileRtol * t) break;
      if (g < 0.0) lo = q; else hi = q;
      // Newton from q when it lands inside the bracket and is under half the previous step, else bisection
      const float step = __fdividef((float)g, (float)f), qn = q - step;
      if (f > 0.0 && qn > lo && qn < hi && fabs(2.0 * g) < fabs((double)dx * f)) {
        dx = step;
        q = qn;
      } else {
        dx = 0.5f * (hi - lo);
        q = lo + dx;
      }
    }
    if (lane == 0) qout[k] = q;
  }

  const float* yp = stage_ptr(p.y.p, st);
  if (!yp) return;
  const float y = yp[(long)b * p.y_stride + p.y_off];
  float* sc = stage_ptr(p.scores.p, st) + (long)b * 3;
  if (isnan(y)) {
    if (lane < 3) sc[lane] = NAN;
    return;
  }
  // CRPS = E|X - y| - E|X - X'| / 2 (Grimit et al. 2006): the component sum, then the pairs s < t of the M^2 pair sum
  // (symmetric) and its diagonal A(0, 2 sigma_s^2) = 2 sigma_s / sqrt(pi).  Log score by log-sum-exp in fp64, PIT = F(y).
  double a_y = 0.0, diag = 0.0, pit = 0.0;
  float lmax = -INFINITY;
  for (int s = lane; s < M; s += 32) {
    const float inv = rsqrtf(v[s]);
    a_y += (double)abs_moment(mu[s] - y, v[s]);
    diag += (double)(v[s] * inv);
    pit += (double)(0.5f * erfcf(-((y - mu[s]) * inv) * kInvSqrt2));
    lmax = fmaxf(lmax, (float)log_kernel(y, mu[s], v[s]));
  }
  lmax = warp_max(lmax);
  double lse = 0.0;
  for (int s = lane; s < M; s += 32) lse += exp(log_kernel(y, mu[s], v[s]) - (double)lmax);
  double pairs = 0.0;
  for (int s = 0; s + 1 < M; ++s) {
    const float ms = mu[s], vs = v[s];
    for (int t = s + 1 + lane; t < M; t += 32) pairs += (double)abs_moment(ms - mu[t], vs + v[t]);
  }
  a_y = warp_sum(a_y);
  diag = warp_sum(diag);
  pit = warp_sum(pit);
  lse = warp_sum(lse);
  pairs = warp_sum(pairs);
  if (lane == 0) {
    sc[0] = (float)(a_y * inv_m - 0.5 * inv_m * inv_m * (2.0 * kInvSqrtPi * diag + 2.0 * pairs));
    sc[1] = (float)(-((double)lmax + log(lse * inv_m)) + kLogSqrt2Pi);
    sc[2] = (float)(pit * inv_m);
  }
}

}  // namespace

int dist_gather(cudaStream_t s, int n_stages, int B, int TO, long off, int64_t r0, int n, int samples,
                const ChainPtrs& pred, const ChainPtrs& var, const ChainPtrs& mu, const ChainPtrs& v) {
  dim3 grid((n + kGatherThreads - 1) / kGatherThreads, n_stages);
  dist_gather_kernel<<<grid, kGatherThreads, 0, s>>>(B, TO, off, r0, n, samples, pred, var, mu, v);
  LFMQ_LAUNCH_CHECK();
  return 0;
}

int mixture_dist(cudaStream_t s, int n_stages, int B, int samples, const float* levels, int n_levels,
                 const ChainPtrs& mu, const ChainPtrs& v, const ChainCPtrs& y, long y_stride, long y_off,
                 const ChainPtrs& quantiles, const ChainPtrs& scores) {
  DistParams p{};
  for (int i = 0; i < n_stages; ++i) {
    p.mu.p[i] = mu.p[i];
    p.v.p[i] = v.p[i];
  }
  p.y = y;
  p.q = quantiles;
  p.scores = scores;
  for (int k = 0; k < n_levels; ++k) p.levels[k] = levels[k];
  p.B = B;
  p.M = samples;
  p.inv_m = 1.0 / samples;
  p.Q = n_levels;
  p.y_stride = y_stride;
  p.y_off = y_off;
  dim3 grid((B + kDistWarps - 1) / kDistWarps, n_stages);
  dist_kernel<<<grid, kDistWarps * 32, 0, s>>>(p);
  LFMQ_LAUNCH_CHECK();
  return 0;
}

}  // namespace lfmq
