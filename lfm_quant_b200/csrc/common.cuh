// Shared helpers for the lfmq CUDA library (sm_90a).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>

#include <atomic>

namespace lfmq {

extern thread_local char g_err[512];
extern std::atomic<long long> g_launches;   // handles may launch from several host threads at once

#define LFMQ_SET_ERR(...) snprintf(::lfmq::g_err, sizeof(::lfmq::g_err), __VA_ARGS__)

#define LFMQ_CUDA_CHECK(expr)                                                              \
  do {                                                                                     \
    cudaError_t _e = (expr);                                                               \
    if (_e != cudaSuccess) {                                                               \
      LFMQ_SET_ERR("%s:%d: %s -> %s", __FILE__, __LINE__, #expr, cudaGetErrorString(_e));  \
      return 2; /* LFMQ_ERR_CUDA */                                                        \
    }                                                                                      \
  } while (0)

// SMs of the current device (grid sizes of the one-wave kernels and of the per-SM partial buffers).
inline int device_sm_count() {
  static const int count = [] {
    int dev = 0, n = 0;
    if (cudaGetDevice(&dev) != cudaSuccess || cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess ||
        n < 1)
      n = 132;
    return n;
  }();
  return count;
}

// Programmatic dependent launch.  Device side: every kernel launched through launch_pdl() calls pdl_sync() before it
// touches anything its predecessors wrote -- wait for the previous kernel of the stream, THEN let the next one's CTAs be
// dispatched (in that order: when a kernel starts, its predecessor has seen ITS predecessor complete, so only the
// immediate predecessor can still be running).  A kernel launched without the attribute sees both as no-ops.
__device__ __forceinline__ void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }
__device__ __forceinline__ void pdl_release() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }
__device__ __forceinline__ void pdl_sync() {
  pdl_wait();
  pdl_release();
}

// Every kernel launch goes through this so bench.py can report gpu_launches.
// LFMQ_DEBUG_SYNC=1: synchronise after every launch and say where (finds the kernel that hangs or faults).
inline bool debug_sync_on() {
  static const bool on = getenv("LFMQ_DEBUG_SYNC") && atoi(getenv("LFMQ_DEBUG_SYNC")) != 0;
  return on;
}
#define LFMQ_DEBUG_SYNC()                                                                              \
  do {                                                                                                 \
    if (::lfmq::debug_sync_on()) {                                                                     \
      fprintf(stderr, "[lfmq launch] %s:%d ...", __FILE__, __LINE__);                                  \
      fflush(stderr);                                                                                  \
      cudaError_t _e = cudaDeviceSynchronize();                                                        \
      fprintf(stderr, " %s\n", cudaGetErrorString(_e));                                               \
      fflush(stderr);                                                                                  \
    }                                                                                                  \
  } while (0)

#define LFMQ_LAUNCH_CHECK()                                   \
  do {                                                        \
    ::lfmq::g_launches++;                                     \
    LFMQ_CUDA_CHECK(cudaGetLastError());                      \
    LFMQ_DEBUG_SYNC();                                        \
  } while (0)

// Host side: launch with the programmatic-stream-serialization attribute when `pdl` is set (LFMQ_PDL=0 turns it off for
// every launch).  `pdl` is per call because a kernel that reads anything before its pdl_wait() must not overlap a
// predecessor that writes it.  `cluster_x` > 1 adds the cluster dimension of the cluster kernels.
template <typename... KArgs, typename... Args>
inline int launch_pdl(void (*kernel)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t s, int cluster_x,
                      bool pdl, Args&&... args) {
  static const bool on = !(getenv("LFMQ_PDL") && atoi(getenv("LFMQ_PDL")) == 0);
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = grid;
  cfg.blockDim = block;
  cfg.dynamicSmemBytes = smem;
  cfg.stream = s;
  cudaLaunchAttribute attr[2];
  int n = 0;
  if (cluster_x > 1) {
    attr[n].id = cudaLaunchAttributeClusterDimension;
    attr[n].val.clusterDim.x = cluster_x;
    attr[n].val.clusterDim.y = 1;
    attr[n].val.clusterDim.z = 1;
    ++n;
  }
  if (on && pdl) {
    attr[n].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[n].val.programmaticStreamSerializationAllowed = 1;
    ++n;
  }
  cfg.attrs = attr;
  cfg.numAttrs = n;
  LFMQ_CUDA_CHECK(cudaLaunchKernelEx(&cfg, kernel, static_cast<KArgs>(args)...));
  g_launches++;
  LFMQ_DEBUG_SYNC();
  return 0;
}

// ---------------------------------------------------------------------------------------------
// Philox4x32-10 (Salmon et al. 2011) -- bit-identical to oracle/lfm_oracle.py:philox4x32_10.
// ---------------------------------------------------------------------------------------------
__host__ __device__ __forceinline__ void philox4x32_10(uint32_t c0, uint32_t c1, uint32_t c2, uint32_t c3,
                                                       uint32_t k0, uint32_t k1, uint32_t out[4]) {
#pragma unroll
  for (int r = 0; r < 10; ++r) {
    const uint64_t p0 = (uint64_t)0xD2511F53u * c0;
    const uint64_t p1 = (uint64_t)0xCD9E8D57u * c2;
    const uint32_t n0 = (uint32_t)(p1 >> 32) ^ c1 ^ k0;
    const uint32_t n1 = (uint32_t)p1;
    const uint32_t n2 = (uint32_t)(p0 >> 32) ^ c3 ^ k1;
    const uint32_t n3 = (uint32_t)p0;
    c0 = n0; c1 = n1; c2 = n2; c3 = n3;
    k0 += 0x9E3779B9u;
    k1 += 0xBB67AE85u;
  }
  out[0] = c0; out[1] = c1; out[2] = c2; out[3] = c3;
}

// Dropout scale factors for the 4 consecutive elements of quad q = (global_row * inner + j) / 4.
struct DropoutKey {
  uint32_t k0, k1;     // seed
  uint32_t stream;     // 2*layer (Dropout) or 2*layer+1 (recurrent dropout)
  uint32_t step;
  uint32_t thr;        // keep iff (r >> 8) >= thr, thr = (uint32)(rate * 2^24)
  float scale;         // 1 / (1 - rate)
};

inline DropoutKey dropout_key(uint64_t seed, int stream, int64_t step, float rate) {
  DropoutKey k;
  k.k0 = (uint32_t)(seed & 0xffffffffu);
  k.k1 = (uint32_t)(seed >> 32);
  k.stream = (uint32_t)stream;
  k.step = (uint32_t)(step & 0xffffffff);
  k.thr = (uint32_t)((double)rate * 16777216.0);
  k.scale = 1.0f / (1.0f - rate);
  return k;
}

__device__ __forceinline__ void dropout_quad(const DropoutKey& k, uint64_t q, float m[4]) {
  uint32_t r[4];
  philox4x32_10((uint32_t)q, (uint32_t)(q >> 32), k.stream, k.step, k.k0, k.k1, r);
#pragma unroll
  for (int i = 0; i < 4; ++i) m[i] = ((r[i] >> 8) >= k.thr) ? k.scale : 0.0f;
}

// softplus of the variance head (custom_layers.py:12-13), shared by the SIMT and tensor-core heads
__device__ __forceinline__ float softplus_f(float a) { return fmaxf(a, 0.f) + log1pf(expf(-fabsf(a))); }

// Carves the caller's workspace into buffers on `granule`-byte boundaries (the handle workspace's 1024 by default);
// with base == nullptr it only sizes.
constexpr size_t WS_ALIGN = 1024;
inline size_t ws_align_up(size_t v) { return (v + WS_ALIGN - 1) / WS_ALIGN * WS_ALIGN; }
struct Carver {
  char* base;
  size_t off;
  size_t granule = WS_ALIGN;
  template <typename T>
  T* take(size_t n) {
    T* p = base ? reinterpret_cast<T*>(base + off) : nullptr;
    off = (off + n * sizeof(T) + granule - 1) / granule * granule;
    return p;
  }
};

// Event brackets around the regions of a step (include/lfmq.h LFMQ_REGION_*).
struct Profiler {
  static constexpr int kRegions = 5, kCap = 256;
  bool enabled = false;
  bool created = false;
  cudaEvent_t a[kRegions][kCap], b[kRegions][kCap];
  int n[kRegions] = {0, 0, 0, 0, 0};
  void begin(int r, cudaStream_t s) {
    if (enabled && n[r] < kCap) cudaEventRecord(a[r][n[r]], s);
  }
  void end(int r, cudaStream_t s) {
    if (enabled && n[r] < kCap) cudaEventRecord(b[r][n[r]++], s);
  }
};

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

__device__ __forceinline__ double warp_sum(double v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// Dropout scale factors of hidden units 8c .. 8c+7 of global row `grow` at step t: quads 2c and 2c+1 of the row's H/4,
// the quads the oracle draws for them.  All ones when `on` is false.
__device__ __forceinline__ void dropout8(const DropoutKey& key, bool on, int64_t grow, int t, int T, int H, int c,
                                         float m[8]) {
  if (on) {
    const uint64_t q = ((uint64_t)grow * T + t) * (uint64_t)(H / 4) + c * 2;
    dropout_quad(key, q, m);
    dropout_quad(key, q + 1, m + 4);
  } else {
#pragma unroll
    for (int e = 0; e < 8; ++e) m[e] = 1.f;
  }
}

// Fixed-order sum of the n partials p[0], p[stride], ..., p[(n-1) stride]: lanes stride over them in fp64, then
// warp_sum.  Deterministic; every lane returns the sum.
template <typename T>
__device__ __forceinline__ double sum_partials(const T* __restrict__ p, long stride, int n) {
  double s = 0.0;
  for (int c = threadIdx.x & 31; c < n; c += 32) s += p[(long)c * stride];
  return warp_sum(s);
}

// ---------------------------------------------------------------------------------------------
// Weighted loss of the point estimate and of RNNUqRangeEstimate (model_utils/losses.py:55-135, 180-284):
//   loss = p1 x0 + (1 - p1) (p2 x1 + (1 - p2) x2)
// x0: mean over the last step's target column, x1: mean over the last step, x2: mean over every unmasked row.
// ---------------------------------------------------------------------------------------------
// A row is masked when all its targets are zero (losses.py:72).
__device__ __forceinline__ bool row_mask(const float* y, int n) {
  bool any = false;
  for (int k = 0; k < n; ++k) any |= (y[k] != 0.0f);
  return any;
}

// Row weights (lfmq_set_row_weights, DESIGN.md section 6d): window b of a training batch weighs w[b] in every sum of the
// loss and in every count a mean divides by; without them (w == nullptr) every window weighs 1.  b is the batch's own
// row, not shifted by row0.  The mask multiplies in: the counts are sums of row_weight * row_mask.
__device__ __forceinline__ float row_weight(const float* w, long b) { return w ? w[b] : 1.f; }

// A weighted count of 0 (every window of the batch weighs 0) divides as 1: its numerators are 0 too, so the loss and
// every gradient are 0.  Unweighted counts are used as they are.
__device__ __forceinline__ float loss_denom(const float* w, float d) { return (w && d == 0.f) ? 1.f : d; }

// dLoss/d(term) of one element of each mean: denom_all and denom_last count the rows the means over every row and over
// the last step divide by; w: the batch's row weights (nullable).
struct LossWeights {
  float all, last, tar;
};
__device__ __forceinline__ LossWeights loss_weights(float p1, float p2, int O, float denom_all, float denom_last,
                                                    const float* w) {
  denom_all = loss_denom(w, denom_all);
  denom_last = loss_denom(w, denom_last);
  return {(1.f - p1) * (1.f - p2) / ((float)O * denom_all), (1.f - p1) * p2 / (denom_last * (float)O), p1 / denom_last};
}

// The squared-error terms of one row of predictions pr (masked by m) against targets y, times the row's weight rw: adds
// them to s0 (last step, column tidx), s1 (last step) and s2 (every column), and with `train` writes dLoss/dpred to dp.
// NCOL > 0: the row is NCOL padded registers, and columns >= O and rows that are not valid contribute exactly zero;
// NCOL = 0: O columns.  The weight scales the first factor of each product (d rw * d, 2 (d rw) ...): rw = 1 leaves every
// operand, and so every rounding and every contraction into an FMA, as it is without weights.
template <int NCOL, typename Acc>
__device__ __forceinline__ void point_loss_row(const float* pr, const float* y, int O, bool valid, float m, float rw,
                                               bool last, int tidx, const LossWeights& w, bool train, float* dp,
                                               Acc& s0, Acc& s1, Acc& s2) {
#pragma unroll
  for (int k = 0; k < (NCOL > 0 ? NCOL : O); ++k) {
    const float d = (k < O && valid) ? (pr[k] * m - y[k]) : 0.f;  // losses.py:75: masked predictions are zeroed
    const float dw = d * rw;
    const float d2 = dw * d;
    s2 += d2;
    float coef = w.all;
    if (last) {
      s1 += d2;
      coef += w.last;
      if (k == tidx) {
        s0 += d2;
        coef += w.tar;
      }
    }
    if (train) dp[k] = 2.f * dw * coef * m;
  }
}

__device__ __forceinline__ double weighted_loss(double p1, double p2, double x0, double x1, double x2) {
  return p1 * x0 + (1.0 - p1) * (p2 * x1 + (1.0 - p2) * x2);
}

// The tensor-core heads keep s0 s1 s2 in three consecutive slots of a [value][cta] partial array.  The warp of the first
// slot, whose sum s0 it holds, sums the other two and writes {loss, mse_0} with the batch denominators {B, unmasked
// rows} (losses.py:87-98), or their weighted sums when the batch has row weights rw.
__device__ __forceinline__ void point_loss_final(const float* __restrict__ slot0, int n_cta, double s0,
                                                 const float* denom, const float* rw, int O, float p1, float p2,
                                                 float* out2) {
  const double s1 = sum_partials(slot0 + n_cta, 1, n_cta);
  const double s2 = sum_partials(slot0 + 2L * n_cta, 1, n_cta);
  if ((threadIdx.x & 31) == 0 && out2) {
    const double Bg = loss_denom(rw, denom[0]), Mg = loss_denom(rw, denom[1]);
    const double mse0 = s0 / Bg, mse1 = s1 / (Bg * O), mse2 = s2 / (Mg * O);
    out2[0] = (float)weighted_loss(p1, p2, mse0, mse1, mse2);
    out2[1] = (float)mse0;
  }
}

// End of a head kernel: each warp's sums of s0 s1 s2 and, with `train`, of the N columns of dLoss/dpred are added
// into the CTA's partial row red_s at loss_at (three slots) and dbo_at (N slots).
template <int N>
__device__ __forceinline__ void flush_loss_sums(float* red_s, int loss_at, int dbo_at, float s0, float s1, float s2,
                                                float (&dbo)[N], bool train) {
  s0 = warp_sum(s0); s1 = warp_sum(s1); s2 = warp_sum(s2);
#pragma unroll
  for (int k = 0; k < N; ++k) dbo[k] = warp_sum(dbo[k]);
  if ((threadIdx.x & 31) == 0) {
    atomicAdd(&red_s[loss_at + 0], s0);
    atomicAdd(&red_s[loss_at + 1], s1);
    atomicAdd(&red_s[loss_at + 2], s2);
    if (train)
      for (int k = 0; k < N; ++k) atomicAdd(&red_s[dbo_at + k], dbo[k]);
  }
}

}  // namespace lfmq
