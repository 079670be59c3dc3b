// fp32 SIMT kernels: the parity path (LFMQ_PREC_FP32) and every HBM-bound piece of the step
// (batcher gather, BN/dropout, head + loss, clip + optimizer + MaxNorm).  sm_90a.
//
// Reference call sites are cited per kernel (paths relative to /root/reference/scripts).
#include "kernels.h"

#include <math.h>

namespace lfmq {

thread_local char g_err[512] = {0};
long long g_launches = 0;

static inline int cdiv(long a, long b) { return (int)((a + b - 1) / b); }

// =============================================================================================
// Generic strided SGEMM, 64x64x16 tiles, 4x4 micro-tiles, deterministic split-K.
// =============================================================================================
constexpr int BM = 64, BN = 64, BK = 16;

template <bool A_M_CONTIG, bool B_N_CONTIG>
__global__ void __launch_bounds__(256) sgemm_kernel(int M, int N, int K, const float* __restrict__ A, long sAm,
                                                    long sAk, const float* __restrict__ B, long sBk, long sBn,
                                                    float* __restrict__ C, long ldc, float beta, int kchunk,
                                                    float* __restrict__ partial) {
  __shared__ __align__(16) float As[BK][BM + 4];
  __shared__ __align__(16) float Bs[BK][BN + 4];
  const int tid = threadIdx.x;
  const int tx = tid & 15, ty = tid >> 4;
  const int m0 = blockIdx.y * BM, n0 = blockIdx.x * BN;
  const int kbeg = blockIdx.z * kchunk;
  const int kend = min(K, kbeg + kchunk);
  float acc[4][4];
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) acc[i][j] = 0.f;

  for (int k0 = kbeg; k0 < kend; k0 += BK) {
#pragma unroll
    for (int r = 0; r < 4; ++r) {
      const int idx = tid + 256 * r;
      int m, k;
      if (A_M_CONTIG) { m = idx & 63; k = idx >> 6; } else { k = idx & 15; m = idx >> 4; }
      const int gm = m0 + m, gk = k0 + k;
      As[k][m] = (gm < M && gk < kend) ? __ldg(A + (long)gm * sAm + (long)gk * sAk) : 0.f;
      int n, kb;
      if (B_N_CONTIG) { n = idx & 63; kb = idx >> 6; } else { kb = idx & 15; n = idx >> 4; }
      const int gn = n0 + n, gkb = k0 + kb;
      Bs[kb][n] = (gn < N && gkb < kend) ? __ldg(B + (long)gkb * sBk + (long)gn * sBn) : 0.f;
    }
    __syncthreads();
#pragma unroll
    for (int k = 0; k < BK; ++k) {
      const float4 a = *reinterpret_cast<const float4*>(&As[k][ty * 4]);
      const float4 b = *reinterpret_cast<const float4*>(&Bs[k][tx * 4]);
      const float av[4] = {a.x, a.y, a.z, a.w};
      const float bv[4] = {b.x, b.y, b.z, b.w};
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[i][j] = fmaf(av[i], bv[j], acc[i][j]);
    }
    __syncthreads();
  }
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int gm = m0 + ty * 4 + i;
    if (gm >= M) continue;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int gn = n0 + tx * 4 + j;
      if (gn >= N) continue;
      if (partial) {
        partial[((long)blockIdx.z * M + gm) * N + gn] = acc[i][j];
      } else {
        float* c = C + (long)gm * ldc + gn;
        *c = (beta == 0.f) ? acc[i][j] : fmaf(beta, *c, acc[i][j]);
      }
    }
  }
}

__global__ void splitk_reduce_kernel(int M, int N, int S, const float* __restrict__ partial, float* __restrict__ C,
                                     long ldc, float beta) {
  const long i = (long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (long)M * N) return;
  float s = 0.f;
  for (int z = 0; z < S; ++z) s += partial[(long)z * M * N + i];
  float* c = C + (i / N) * ldc + (i % N);
  *c = (beta == 0.f) ? s : fmaf(beta, *c, s);
}

int sgemm(cudaStream_t s, int M, int N, int K, const float* A, long sAm, long sAk, const float* B, long sBk,
          long sBn, float* C, long ldc, float beta, float* scratch, size_t scratch_elems) {
  if (M <= 0 || N <= 0) return 0;
  const int tiles = cdiv(M, BM) * cdiv(N, BN);
  int S = 1;
  if (K >= 2048 && tiles < 296 && scratch) {
    S = min(cdiv(K, 512), max(1, 592 / tiles));
    while (S > 1 && (size_t)S * M * N > scratch_elems) --S;
  }
  int kchunk = cdiv(cdiv(K, S), BK) * BK;
  if (kchunk <= 0) kchunk = BK;
  S = max(1, cdiv(K, kchunk));
  dim3 grid(cdiv(N, BN), cdiv(M, BM), S);
  float* partial = (S > 1) ? scratch : nullptr;
  const bool am = (sAm == 1), bn = (sBn == 1);
  if (am && bn)
    sgemm_kernel<true, true><<<grid, 256, 0, s>>>(M, N, K, A, sAm, sAk, B, sBk, sBn, C, ldc, beta, kchunk, partial);
  else if (am && !bn)
    sgemm_kernel<true, false><<<grid, 256, 0, s>>>(M, N, K, A, sAm, sAk, B, sBk, sBn, C, ldc, beta, kchunk, partial);
  else if (!am && bn)
    sgemm_kernel<false, true><<<grid, 256, 0, s>>>(M, N, K, A, sAm, sAk, B, sBk, sBn, C, ldc, beta, kchunk, partial);
  else
    sgemm_kernel<false, false><<<grid, 256, 0, s>>>(M, N, K, A, sAm, sAk, B, sBk, sBn, C, ldc, beta, kchunk, partial);
  LFMQ_LAUNCH_CHECK();
  if (S > 1) {
    splitk_reduce_kernel<<<cdiv((long)M * N, 256), 256, 0, s>>>(M, N, S, partial, C, ldc, beta);
    LFMQ_LAUNCH_CHECK();
  }
  return 0;
}

// =============================================================================================
// LSTM cell, pointwise halves of one time step (Keras LSTM implementation=2,
// models/point_estimate/rnn_point_estimate.py:80-87; SURVEY App. A.1 / A.4).
// =============================================================================================
__device__ __forceinline__ float sigmoid_f(float x) { return 1.0f / (1.0f + expf(-x)); }

__global__ void lstm_pointwise_fwd_kernel(int B, int T, int H, int t, const float* __restrict__ z,
                                          const float* __restrict__ bias, float* __restrict__ gates,
                                          float* __restrict__ c, float* __restrict__ h,
                                          const float* __restrict__ rmask, float* __restrict__ hm) {
  const long idx = (long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= (long)B * H) return;
  const int b = (int)(idx / H), j = (int)(idx % H);
  const float* zr = z + (long)b * 4 * H;
  const float gi = sigmoid_f(zr[j] + bias[j]);
  const float gf = sigmoid_f(zr[H + j] + bias[H + j]);
  const float gg = tanhf(zr[2 * H + j] + bias[2 * H + j]);
  const float go = sigmoid_f(zr[3 * H + j] + bias[3 * H + j]);
  const long o = ((long)b * T + t) * H + j;
  const float cp = (t > 0) ? c[o - H] : 0.f;
  const float cn = fmaf(gf, cp, gi * gg);
  const float hn = go * tanhf(cn);
  c[o] = cn;
  h[o] = hn;
  if (gates) {
    float* g = gates + ((long)b * T + t) * 4 * H;
    g[j] = gi; g[H + j] = gf; g[2 * H + j] = gg; g[3 * H + j] = go;
  }
  if (hm) hm[idx] = rmask ? hn * rmask[idx] : hn;
}

int lstm_pointwise_fwd(cudaStream_t s, int B, int T, int H, int t, const float* z, const float* bias, float* gates,
                       float* c, float* h, const float* rmask, float* hm) {
  lstm_pointwise_fwd_kernel<<<cdiv((long)B * H, 256), 256, 0, s>>>(B, T, H, t, z, bias, gates, c, h, rmask, hm);
  LFMQ_LAUNCH_CHECK();
  return 0;
}

// dz_t from (dh_out_t + dh_rec), saved gates and cell states; dc carried in place.
__global__ void lstm_pointwise_bwd_kernel(int B, int T, int H, int t, const float* __restrict__ gates,
                                          const float* __restrict__ c, const float* __restrict__ dh_out,
                                          const float* __restrict__ dh_rec, const float* __restrict__ rmask,
                                          float* __restrict__ dc, float* __restrict__ dz) {
  const long idx = (long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= (long)B * H) return;
  const int b = (int)(idx / H), j = (int)(idx % H);
  const long o = ((long)b * T + t) * H + j;
  const float* g = gates + ((long)b * T + t) * 4 * H;
  const float gi = g[j], gf = g[H + j], gg = g[2 * H + j], go = g[3 * H + j];
  float dh = dh_out[o];
  if (dh_rec) dh += rmask ? dh_rec[idx] * rmask[idx] : dh_rec[idx];
  const float tc = tanhf(c[o]);
  const float cp = (t > 0) ? c[o - H] : 0.f;
  const float d_o = dh * tc;
  const float dcn = ((t < T - 1) ? dc[idx] : 0.f) + dh * go * (1.f - tc * tc);
  const float di = dcn * gg, dg = dcn * gi, df = dcn * cp;
  dc[idx] = dcn * gf;
  float* d = dz + ((long)b * T + t) * 4 * H;
  d[j] = di * gi * (1.f - gi);
  d[H + j] = df * gf * (1.f - gf);
  d[2 * H + j] = dg * (1.f - gg * gg);
  d[3 * H + j] = d_o * go * (1.f - go);
}

int lstm_pointwise_bwd(cudaStream_t s, int B, int T, int H, int t, const float* gates, const float* c,
                       const float* dh_out, const float* dh_rec, const float* rmask, float* dc, float* dz) {
  lstm_pointwise_bwd_kernel<<<cdiv((long)B * H, 256), 256, 0, s>>>(B, T, H, t, gates, c, dh_out, dh_rec, rmask, dc,
                                                                   dz);
  LFMQ_LAUNCH_CHECK();
  return 0;
}

// =============================================================================================
// GRU cell (Keras GRU, reset_after=True, implementation=2; rnn_point_estimate.py:89-98), pointwise halves of one step.
//   zx = x_t W  [B,3H]   zh = (h_{t-1} * mask) U  [B,3H] (absent at t = 0)   bias [2][3H] = input row | recurrent row
//   z = sig(zx_z + zh_z + b), r = sig(zx_r + zh_r + b), q = zh_h + b_rh, hh = tanh(zx_h + b_ih + r q)
//   h_t = z h_{t-1} + (1 - z) hh.   Saved per step (same 4H slot as the LSTM gates): z | r | hh | q.
// =============================================================================================
__global__ void gru_pointwise_fwd_kernel(int B, int T, int H, int t, const float* __restrict__ zx,
                                         const float* __restrict__ zh, const float* __restrict__ bias,
                                         float* __restrict__ gates, float* __restrict__ h,
                                         const float* __restrict__ rmask, float* __restrict__ hm) {
  const long idx = (long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= (long)B * H) return;
  const int b = (int)(idx / H), j = (int)(idx % H);
  const float* xr = zx + (long)b * 3 * H;
  const float* bi = bias;
  const float* br = bias + 3 * H;
  float hz = br[j], hr = br[H + j], q = br[2 * H + j];
  if (zh) {
    const float* hrw = zh + (long)b * 3 * H;
    hz += hrw[j]; hr += hrw[H + j]; q += hrw[2 * H + j];
  }
  const float gz = sigmoid_f(xr[j] + bi[j] + hz);
  const float gr = sigmoid_f(xr[H + j] + bi[H + j] + hr);
  const float hh = tanhf(xr[2 * H + j] + bi[2 * H + j] + gr * q);
  const long o = ((long)b * T + t) * H + j;
  const float hp = (t > 0) ? h[o - H] : 0.f;
  const float hn = fmaf(gz, hp - hh, hh);
  h[o] = hn;
  if (gates) {
    float* g = gates + ((long)b * T + t) * 4 * H;
    g[j] = gz; g[H + j] = gr; g[2 * H + j] = hh; g[3 * H + j] = q;
  }
  if (hm) hm[idx] = rmask ? hn * rmask[idx] : hn;
}

int gru_pointwise_fwd(cudaStream_t s, int B, int T, int H, int t, const float* zx, const float* zh, const float* bias,
                      float* gates, float* h, const float* rmask, float* hm) {
  gru_pointwise_fwd_kernel<<<cdiv((long)B * H, 256), 256, 0, s>>>(B, T, H, t, zx, zh, bias, gates, h, rmask, hm);
  LFMQ_LAUNCH_CHECK();
  return 0;
}

// Gradients w.r.t. the input projection (dxz) and the recurrent projection (dhz) of step t; the part of dLoss/dh that
// reaches h_{t-1} through z * h_{t-1} is carried in place in `dcarry`.
__global__ void gru_pointwise_bwd_kernel(int B, int T, int H, int t, const float* __restrict__ gates,
                                         const float* __restrict__ h, const float* __restrict__ dh_out,
                                         const float* __restrict__ dh_rec, const float* __restrict__ rmask,
                                         float* __restrict__ dcarry, float* __restrict__ dxz,
                                         float* __restrict__ dhz) {
  const long idx = (long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= (long)B * H) return;
  const int b = (int)(idx / H), j = (int)(idx % H);
  const long o = ((long)b * T + t) * H + j;
  const float* g = gates + ((long)b * T + t) * 4 * H;
  const float gz = g[j], gr = g[H + j], hh = g[2 * H + j], q = g[3 * H + j];
  float dh = dh_out[o];
  if (t < T - 1) dh += dcarry[idx];
  if (dh_rec) dh += rmask ? dh_rec[idx] * rmask[idx] : dh_rec[idx];
  const float hp = (t > 0) ? h[o - H] : 0.f;
  const float da_h = dh * (1.f - gz) * (1.f - hh * hh);
  const float da_z = dh * (hp - hh) * gz * (1.f - gz);
  const float da_r = da_h * q * gr * (1.f - gr);
  dcarry[idx] = dh * gz;
  float* dx = dxz + ((long)b * T + t) * 3 * H;
  float* dr = dhz + ((long)b * T + t) * 3 * H;
  dx[j] = da_z; dx[H + j] = da_r; dx[2 * H + j] = da_h;
  dr[j] = da_z; dr[H + j] = da_r; dr[2 * H + j] = da_h * gr;
}

int gru_pointwise_bwd(cudaStream_t s, int B, int T, int H, int t, const float* gates, const float* h,
                      const float* dh_out, const float* dh_rec, const float* rmask, float* dcarry, float* dxz,
                      float* dhz) {
  gru_pointwise_bwd_kernel<<<cdiv((long)B * H, 256), 256, 0, s>>>(B, T, H, t, gates, h, dh_out, dh_rec, rmask, dcarry,
                                                                  dxz, dhz);
  LFMQ_LAUNCH_CHECK();
  return 0;
}

// recurrent_dropout mask [B,H], one per call, shared by all T steps (rnn_point_estimate.py:86).
__global__ void gen_row_mask_kernel(int B, int H, DropoutKey key, int64_t row0, float* __restrict__ rmask) {
  const long q = (long)blockIdx.x * blockDim.x + threadIdx.x;
  const int nq = H / 4;
  if (q >= (long)B * nq) return;
  const long b = q / nq;
  float m[4];
  dropout_quad(key, (uint64_t)(row0 + b) * nq + (q % nq), m);
  *reinterpret_cast<float4*>(rmask + q * 4) = make_float4(m[0], m[1], m[2], m[3]);
}

int gen_row_mask(cudaStream_t s, int B, int H, DropoutKey key, int64_t row0, float* rmask) {
  gen_row_mask_kernel<<<cdiv((long)B * H / 4, 256), 256, 0, s>>>(B, H, key, row0, rmask);
  LFMQ_LAUNCH_CHECK();
  return 0;
}

// hp[b,t,:] = (t > 0 ? h[b,t-1,:] : 0) * rmask[b,:]  -- the operand of dU = hp^T dz (App. A.4).
__global__ void shift_mask_kernel(int B, int T, int H, const float* __restrict__ h, const float* __restrict__ rmask,
                                  float* __restrict__ hp) {
  const long idx = (long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= (long)B * T * H) return;
  const int j = (int)(idx % H);
  const long bt = idx / H;
  const int t = (int)(bt % T);
  const long b = bt / T;
  float v = (t > 0) ? h[idx - H] : 0.f;
  if (rmask) v *= rmask[b * H + j];
  hp[idx] = v;
}

int shift_mask(cudaStream_t s, int B, int T, int H, const float* h, const float* rmask, float* hp) {
  shift_mask_kernel<<<cdiv((long)B * T * H, 256), 256, 0, s>>>(B, T, H, h, rmask, hp);
  LFMQ_LAUNCH_CHECK();
  return 0;
}

// =============================================================================================
// BatchNormalization (inference-mode affine, SURVEY App. B #1) + Dropout
// (rnn_point_estimate.py:88-89).
// =============================================================================================
__global__ void bn_dropout_fwd_kernel(long nquads, int T, int H, const float* __restrict__ h,
                                      const float* __restrict__ gamma, const float* __restrict__ beta,
                                      const float* __restrict__ mean, const float* __restrict__ var, float eps,
                                      bool use_dropout, DropoutKey key, int64_t row0, float* __restrict__ y) {
  const long q = (long)blockIdx.x * blockDim.x + threadIdx.x;
  if (q >= nquads) return;
  const int nq = H / 4;
  const int j = (int)(q % nq) * 4;
  const float4 hv = *reinterpret_cast<const float4*>(h + q * 4);
  float m[4] = {1.f, 1.f, 1.f, 1.f};
  if (use_dropout) dropout_quad(key, (uint64_t)row0 * T * nq + q, m);
  const float hin[4] = {hv.x, hv.y, hv.z, hv.w};
  float out[4];
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const float inv = 1.0f / sqrtf(var[j + i] + eps);
    out[i] = (gamma[j + i] * (hin[i] - mean[j + i]) * inv + beta[j + i]) * m[i];
  }
  *reinterpret_cast<float4*>(y + q * 4) = make_float4(out[0], out[1], out[2], out[3]);
}

int bn_dropout_fwd(cudaStream_t s, int B, int T, int H, const float* h, const float* gamma, const float* beta,
                   const float* mean, const float* var, float eps, bool use_dropout, DropoutKey key, int64_t row0,
                   float* y) {
  const long nquads = (long)B * T * H / 4;
  bn_dropout_fwd_kernel<<<cdiv(nquads, 256), 256, 0, s>>>(nquads, T, H, h, gamma, beta, mean, var, eps, use_dropout,
                                                          key, row0, y);
  LFMQ_LAUNCH_CHECK();
  return 0;
}

// dh_out = dy * d * gamma * inv ; per-block partial column sums of dgamma, dbeta -> scratch[blk][2H].
constexpr int BN_ROWS_PER_BLOCK = 128;

__global__ void bn_dropout_bwd_kernel(long rows, int T, int H, const float* __restrict__ dy,
                                      const float* __restrict__ h, const float* __restrict__ gamma,
                                      const float* __restrict__ mean, const float* __restrict__ var, float eps,
                                      bool use_dropout, DropoutKey key, int64_t row0, float* __restrict__ dh_out,
                                      float* __restrict__ partial) {
  extern __shared__ float red[];  // [RL][2*H]
  const int nq = H / 4;
  const int RL = blockDim.x / nq;
  const int qc = threadIdx.x % nq, rl = threadIdx.x / nq;
  const int j = qc * 4;
  float g[4], mu[4], inv[4], sg[4] = {0, 0, 0, 0}, sb[4] = {0, 0, 0, 0};
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    g[i] = gamma[j + i];
    mu[i] = mean[j + i];
    inv[i] = 1.0f / sqrtf(var[j + i] + eps);
  }
  const long r0 = (long)blockIdx.x * BN_ROWS_PER_BLOCK;
  const long r1 = min(rows, r0 + BN_ROWS_PER_BLOCK);
  if (rl < RL) {
    for (long r = r0 + rl; r < r1; r += RL) {
      const long q = r * nq + qc;
      const float4 dv = *reinterpret_cast<const float4*>(dy + q * 4);
      const float4 hv = *reinterpret_cast<const float4*>(h + q * 4);
      float m[4] = {1.f, 1.f, 1.f, 1.f};
      if (use_dropout) dropout_quad(key, (uint64_t)row0 * T * nq + q, m);
      const float d[4] = {dv.x * m[0], dv.y * m[1], dv.z * m[2], dv.w * m[3]};
      const float hh[4] = {hv.x, hv.y, hv.z, hv.w};
      float o[4];
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        sg[i] += d[i] * (hh[i] - mu[i]) * inv[i];
        sb[i] += d[i];
        o[i] = d[i] * g[i] * inv[i];
      }
      *reinterpret_cast<float4*>(dh_out + q * 4) = make_float4(o[0], o[1], o[2], o[3]);
    }
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      red[(long)rl * 2 * H + j + i] = sg[i];
      red[(long)rl * 2 * H + H + j + i] = sb[i];
    }
  }
  __syncthreads();
  for (int c = threadIdx.x; c < 2 * H; c += blockDim.x) {
    float sum = 0.f;
    for (int r = 0; r < RL; ++r) sum += red[(long)r * 2 * H + c];
    partial[(long)blockIdx.x * 2 * H + c] = sum;
  }
}

__global__ void colsum_partial_kernel(long rows, int N, long rows_per_block, const float* __restrict__ A,
                                      float* __restrict__ partial) {
  const long r0 = (long)blockIdx.x * rows_per_block;
  const long r1 = min(rows, r0 + rows_per_block);
  for (int n = threadIdx.x; n < N; n += blockDim.x) {
    float s = 0.f;
    for (long r = r0; r < r1; ++r) s += A[r * N + n];
    partial[(long)blockIdx.x * N + n] = s;
  }
}

int colsum(cudaStream_t s, long rows, int N, const float* A, float* out, float* scratch, size_t scratch_elems) {
  long nblk = min((long)1024, max((long)1, rows / 64));
  while (nblk > 1 && (size_t)nblk * N > scratch_elems) nblk /= 2;
  if (nblk <= 1) {
    colsum_partial_kernel<<<1, 256, 0, s>>>(rows, N, rows, A, out);
    LFMQ_LAUNCH_CHECK();
    return 0;
  }
  const long rpb = (rows + nblk - 1) / nblk;
  nblk = (rows + rpb - 1) / rpb;
  colsum_partial_kernel<<<(int)nblk, 256, 0, s>>>(rows, N, rpb, A, scratch);
  LFMQ_LAUNCH_CHECK();
  colsum_partial_kernel<<<1, 256, 0, s>>>(nblk, N, nblk, scratch, out);
  LFMQ_LAUNCH_CHECK();
  return 0;
}

int bn_dropout_bwd(cudaStream_t s, int B, int T, int H, const float* dy, const float* h, const float* gamma,
                   const float* mean, const float* var, float eps, bool use_dropout, DropoutKey key, int64_t row0,
                   float* dh_out, float* dgamma, float* dbeta, float* scratch, size_t scratch_elems) {
  if (dbeta != dgamma + H) {
    LFMQ_SET_ERR("bn_dropout_bwd: dgamma/dbeta must be adjacent");
    return 1;
  }
  const long rows = (long)B * T;
  const int nq = H / 4;
  if (nq > 256) {
    LFMQ_SET_ERR("bn_dropout_bwd: num_hidden > 1024 unsupported");
    return 3;
  }
  const int RL = max(1, 256 / nq);
  const int nblk = cdiv(rows, BN_ROWS_PER_BLOCK);
  const size_t need = (size_t)nblk * 2 * H + (size_t)1024 * 2 * H;
  if (need > scratch_elems) {
    LFMQ_SET_ERR("bn_dropout_bwd: scratch too small (%zu > %zu)", need, scratch_elems);
    return 4;
  }
  bn_dropout_bwd_kernel<<<nblk, nq * RL, (size_t)RL * 2 * H * sizeof(float), s>>>(
      rows, T, H, dy, h, gamma, mean, var, eps, use_dropout, key, row0, dh_out, scratch);
  LFMQ_LAUNCH_CHECK();
  return colsum(s, nblk, 2 * H, scratch, dgamma, scratch + (size_t)nblk * 2 * H, (size_t)1024 * 2 * H);
}

__global__ void add_bias_rows_kernel(long n, int N, float* __restrict__ C, const float* __restrict__ bias) {
  const long i = (long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) C[i] += bias[i % N];
}

int add_bias_rows(cudaStream_t s, long rows, int N, float* C, const float* bias) {
  add_bias_rows_kernel<<<cdiv(rows * N, 256), 256, 0, s>>>(rows * N, N, C, bias);
  LFMQ_LAUNCH_CHECK();
  return 0;
}

// ---- window index on the device (data_processing.py:170-305: _create_tf_dataset + _append_sequence_data) -------------
// One thread per table row.  cur_len[i] = i - (start of the row's key run) + 1 (:218-219,227) comes from an inclusive
// max-scan of (key[i] != key[i-1] ? i : 0); the rows that yield a window (:221-234) are compacted in row order by an
// exclusive sum-scan of their flags.  Both scans: per-block scan + one block over the block aggregates.
constexpr int WI_THREADS = 1024;

template <bool MAX>
__device__ __forceinline__ int wi_block_scan(int v, int* total) {      // inclusive scan over the block's 1024 threads
  __shared__ int warp_tot[32];
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const int u = __shfl_up_sync(0xffffffffu, v, o);
    if (lane >= o) v = MAX ? max(v, u) : v + u;
  }
  __syncthreads();                        // warp_tot may still be read by the previous call
  if (lane == 31) warp_tot[w] = v;
  __syncthreads();
  if (w == 0) {
    int t = warp_tot[lane];
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const int u = __shfl_up_sync(0xffffffffu, t, o);
      if (lane >= o) t = MAX ? max(t, u) : t + u;
    }
    warp_tot[lane] = t;
  }
  __syncthreads();
  if (w > 0) v = MAX ? max(v, warp_tot[w - 1]) : v + warp_tot[w - 1];
  if (total) *total = warp_tot[31];
  return v;
}

// pass 1: block aggregate of the run-start candidates
__global__ void __launch_bounds__(WI_THREADS) wi_runstart_agg_kernel(int n, const int32_t* __restrict__ key,
                                                                     int* __restrict__ blk_max) {
  const int i = blockIdx.x * WI_THREADS + threadIdx.x;
  int v = 0;
  if (i < n && i > 0 && key[i] != key[i - 1]) v = i;
  int tot;
  wi_block_scan<true>(v, &tot);
  if (threadIdx.x == 0) blk_max[blockIdx.x] = tot;
}

// one block: exclusive scan of the nb block aggregates (element i combines in[0..i-1]); total (nullable) = all of them.
// Thread k of a chunk loads in[i-1]: the inclusive scan of the shifted input is the exclusive scan.
template <bool MAX>
__global__ void __launch_bounds__(WI_THREADS) wi_scan_aggs_kernel(int nb, const int* __restrict__ in,
                                                                  int* __restrict__ out_excl, int* __restrict__ total) {
  int carry = 0;
  for (int base = 0; base <= nb; base += WI_THREADS) {
    const int i = base + threadIdx.x;
    const int v = (i >= 1 && i <= nb) ? in[i - 1] : 0;
    int tot;
    const int inc = wi_block_scan<MAX>(v, &tot);
    if (i < nb) out_excl[i] = MAX ? max(inc, carry) : inc + carry;
    carry = MAX ? max(carry, tot) : carry + tot;
  }
  if (total && threadIdx.x == 0) *total = carry;
}

// pass 2: cur_len, the window test, per-row (seq_len, flag) and the block's window count
__global__ void __launch_bounds__(WI_THREADS) wi_flags_kernel(WindowIndexArgs a, const int* __restrict__ blk_start_excl,
                                                              int* __restrict__ seq_len_out, int* __restrict__ blk_cnt) {
  const int i = blockIdx.x * WI_THREADS + threadIdx.x;
  int v = 0;
  if (i < a.n && i > 0 && a.key[i] != a.key[i - 1]) v = i;
  int run_start = wi_block_scan<true>(v, nullptr);
  run_start = max(run_start, blk_start_excl[blockIdx.x]);
  int ok = 0, sl = 0;
  if (i < a.n) {
    const int cur_len = i - run_start + 1;
    const int32_t d = a.date[i];
    const bool same_tar = (i + a.forecast_n <= a.n - 1) && a.key[i + a.forecast_n] == a.key[i];       // :213-216
    if (a.train)                                                                                          // :221-225
      ok = cur_len >= a.min_steps && a.active[i] && d >= a.start_date && d <= a.last_train_date && same_tar;
    else                                                                                                  // :231-234
      ok = cur_len >= a.min_steps && a.active[i] && d >= a.start_date && d <= a.end_date;
    sl = min(cur_len - (cur_len - 1) % a.stride, a.max_steps);                                            // :263
    seq_len_out[i] = ok ? sl : 0;
  }
  int tot;
  wi_block_scan<false>(ok, &tot);
  if (threadIdx.x == 0) blk_cnt[blockIdx.x] = tot;
}

// pass 3: compaction in row order
__global__ void __launch_bounds__(WI_THREADS) wi_scatter_kernel(WindowIndexArgs a, const int* __restrict__ seq_len_in,
                                                                const int* __restrict__ blk_off, int cap,
                                                                int32_t* __restrict__ inp, int32_t* __restrict__ tar,
                                                                int32_t* __restrict__ rows) {
  const int i = blockIdx.x * WI_THREADS + threadIdx.x;
  const int sl = i < a.n ? seq_len_in[i] : 0;
  const int ok = sl > 0;
  const int pos = wi_block_scan<false>(ok, nullptr) - ok + blk_off[blockIdx.x];
  if (!ok || pos >= cap) return;
  const int pad = (a.max_steps - sl) / a.stride;                                                          // :264
  const bool same_tar = (i + a.forecast_n <= a.n - 1) && a.key[i + a.forecast_n] == a.key[i];
  inp[3 * pos + 0] = i - sl + 1;
  inp[3 * pos + 1] = i;
  inp[3 * pos + 2] = pad;
  tar[3 * pos + 0] = i - sl + 1 + a.forecast_n;                                                           // :270-279
  tar[3 * pos + 1] = same_tar ? i + a.forecast_n : i;
  tar[3 * pos + 2] = pad;
  rows[pos] = i;
}

int window_index(cudaStream_t s, const WindowIndexArgs& a, int cap, int32_t* inp, int32_t* tar, int32_t* rows,
                 int32_t* count, int* work) {
  const int nb = cdiv(a.n, WI_THREADS);
  int* blk_max = work;                  // [nb]
  int* blk_start = work + nb;           // [nb]
  int* blk_cnt = work + 2 * nb;         // [nb]
  int* blk_off = work + 3 * nb;         // [nb]
  int* seq_len = work + 4 * nb;         // [n]
  wi_runstart_agg_kernel<<<nb, WI_THREADS, 0, s>>>(a.n, a.key, blk_max);
  LFMQ_LAUNCH_CHECK();
  wi_scan_aggs_kernel<true><<<1, WI_THREADS, 0, s>>>(nb, blk_max, blk_start, nullptr);
  LFMQ_LAUNCH_CHECK();
  wi_flags_kernel<<<nb, WI_THREADS, 0, s>>>(a, blk_start, seq_len, blk_cnt);
  LFMQ_LAUNCH_CHECK();
  wi_scan_aggs_kernel<false><<<1, WI_THREADS, 0, s>>>(nb, blk_cnt, blk_off, count);
  LFMQ_LAUNCH_CHECK();
  wi_scatter_kernel<<<nb, WI_THREADS, 0, s>>>(a, seq_len, blk_off, cap, inp, tar, rows);
  LFMQ_LAUNCH_CHECK();
  return 0;
}

// ---- forecast_steps > 1: glue between the stages (rnn_point_estimate.py:109-124; model_base_class.py:18-51) ----
// next[b, t, :] = prev[b, t + 1, :] for t < T-1 (Cropping1D((1,0)) of the concatenation), and the appended step
// next[b, T-1, :] = [pred[b, T-1, 0:O], x0[b, T-1, O:F]] (latest prediction + the last AVAILABLE aux features).
__global__ void chain_next_input_kernel(long n, int T, int F, int O, const float* __restrict__ prev,
                                        const float* __restrict__ pred, const float* __restrict__ x0,
                                        float* __restrict__ next) {
  const long i = (long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const int k = (int)(i % F);
  const long bt = i / F;
  const int t = (int)(bt % T);
  const long b = bt / T;
  float v;
  if (t < T - 1) v = prev[i + F];
  else if (k < O) v = pred[(b * T + (T - 1)) * O + k];
  else v = x0[i];
  next[i] = v;
}

int chain_next_input(cudaStream_t s, int B, int T, int F, int O, const float* prev, const float* pred, const float* x0,
                     float* next) {
  const long n = (long)B * T * F;
  chain_next_input_kernel<<<cdiv(n, 256), 256, 0, s>>>(n, T, F, O, prev, pred, x0, next);
  LFMQ_LAUNCH_CHECK();
  return 0;
}

__global__ void scale_inplace_kernel(long n, float* __restrict__ p, float w) {
  const long i = (long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) p[i] *= w;
}

int scale_inplace(cudaStream_t s, long n, float* p, float w) {
  scale_inplace_kernel<<<cdiv(n, 256), 256, 0, s>>>(n, p, w);
  LFMQ_LAUNCH_CHECK();
  return 0;
}

// The input window of stage `stage` holds, at time position T-1-j (j = 0..stage-1), the step appended for stage
// stage-j, whose first O columns are pred_{stage-1-j}[:, T-1, :]: the input gradient flows back into those rows.
__global__ void chain_scatter_dx_kernel(int B, int T, int F, int O, int stage, const float* __restrict__ dx,
                                        ChainPtrs dpred) {
  const long i = (long)blockIdx.x * blockDim.x + threadIdx.x;
  const long n = (long)B * stage * O;
  if (i >= n) return;
  const int k = (int)(i % O);
  const int j = (int)((i / O) % stage);
  const long b = i / ((long)O * stage);
  dpred.p[stage - 1 - j][(b * T + (T - 1)) * O + k] += dx[(b * T + (T - 1 - j)) * F + k];
}

int chain_scatter_dx(cudaStream_t s, int B, int T, int F, int O, int stage, const float* dx, const ChainPtrs& dpred) {
  const long n = (long)B * stage * O;
  chain_scatter_dx_kernel<<<cdiv(n, 256), 256, 0, s>>>(B, T, F, O, stage, dx, dpred);
  LFMQ_LAUNCH_CHECK();
  return 0;
}

// tf.clip_by_global_norm over ALL stages' variables (train.py:196): every stage's tail holds its own ||g||; this
// writes the joint norm and the joint clip scale into each of them.  out2 (nullable) = sum_s w_s {loss_s, mse_s}
// (Losses.weight_adjusted_mse, losses.py:47-51), read from the stages' {loss, mse_0} pairs.
__global__ void chain_combine_kernel(int S, ChainPtrs scalars, float clip, ChainPtrs loss2, ChainWeights w,
                                     float* __restrict__ out2) {
  if (threadIdx.x != 0 || blockIdx.x != 0) return;
  if (scalars.p[0]) {
    double ss = 0;
    for (int s = 0; s < S; ++s) ss += (double)scalars.p[s][0] * (double)scalars.p[s][0];
    const float gn = (float)sqrt(ss);
    const float sc = (clip > 0.f) ? clip / fmaxf(gn, clip) : 1.0f;
    for (int s = 0; s < S; ++s) {
      scalars.p[s][0] = gn;
      scalars.p[s][1] = sc;
    }
  }
  if (out2) {
    float l = 0.f, m = 0.f;
    for (int s = 0; s < S; ++s) {
      l += w.w[s] * loss2.p[s][0];
      m += w.w[s] * loss2.p[s][1];
    }
    out2[0] = l;
    out2[1] = m;
  }
}

int chain_combine(cudaStream_t s, int S, const ChainPtrs& scalars, float clip, const ChainPtrs& loss2,
                  const ChainWeights& w, float* out2) {
  chain_combine_kernel<<<1, 32, 0, s>>>(S, scalars, clip, loss2, w, out2);
  LFMQ_LAUNCH_CHECK();
  return 0;
}

__global__ void fill_kernel(float* p, long n, float v) {
  const long i = (long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) p[i] = v;
}

int fill(cudaStream_t s, float* p, long n, float v) {
  if (n <= 0) return 0;
  fill_kernel<<<cdiv(n, 256), 256, 0, s>>>(p, n, v);
  LFMQ_LAUNCH_CHECK();
  return 0;
}

// =============================================================================================
// Loss (model_utils/losses.py:55-98,121-135; SURVEY App. A.3), one thread per [b,t] row.
// =============================================================================================
constexpr int LOSS_BLOCKS = 296;

__device__ __forceinline__ void block_reduce4(double v[4], double* out4) {
  __shared__ double sm[4][8];
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    v[i] = warp_sum(v[i]);
    if (lane == 0) sm[i][w] = v[i];
  }
  __syncthreads();
  if (threadIdx.x < 4) {
    double s = 0;
    for (int k = 0; k < (int)(blockDim.x >> 5); ++k) s += sm[threadIdx.x][k];
    out4[threadIdx.x] = s;
  }
}

__global__ void __launch_bounds__(256) loss_rows_kernel(int B, int T, int O, const float* __restrict__ pred,
                                                        const float* __restrict__ y,
                                                        const float* __restrict__ denom, int target_idx, float p1,
                                                        float p2, float* __restrict__ dpred,
                                                        double* __restrict__ partial) {
  double acc[4] = {0, 0, 0, 0};  // s0, s1, s2, mask count
  float c_all = 0.f, c_last = 0.f, c_tar = 0.f;
  if (dpred) {
    const float Bg = denom[0], Mg = denom[1];
    c_all = (1.f - p1) * (1.f - p2) / ((float)O * Mg);
    c_last = (1.f - p1) * p2 / (Bg * (float)O);
    c_tar = p1 / Bg;
  }
  const long rows = (long)B * T;
  for (long r = (long)blockIdx.x * blockDim.x + threadIdx.x; r < rows; r += (long)gridDim.x * blockDim.x) {
    const float* yr = y + r * O;
    const float* pr = pred ? pred + r * O : nullptr;
    bool any = false;
    for (int k = 0; k < O; ++k) any |= (yr[k] != 0.0f);          // losses.py:72
    const float m = any ? 1.f : 0.f;
    acc[3] += m;
    if (!pr) continue;
    const bool last = ((int)(r % T) == T - 1);
    for (int k = 0; k < O; ++k) {
      const float d = pr[k] * m - yr[k];                           // losses.py:75
      const float d2 = d * d;
      acc[2] += d2;
      float coef = c_all;
      if (last) {
        acc[1] += d2;
        coef += c_last;
        if (k == target_idx) { acc[0] += d2; coef += c_tar; }
      }
      if (dpred) dpred[r * O + k] = 2.f * d * coef * m;
    }
  }
  block_reduce4(acc, partial + (long)blockIdx.x * 4);
}

// mode 0: maskout = {B, mask_count};  mode 1: out = {loss, mse_0} (+ maskout when given)
__global__ void loss_final_kernel(int nblk, const double* __restrict__ partial, const float* __restrict__ denom,
                                  int B, int O, float p1, float p2, int mode, float* __restrict__ out,
                                  float* __restrict__ maskout) {
  // one warp, fixed summation order (lane-strided then butterfly): deterministic
  double s[4] = {0, 0, 0, 0};
  for (int b = threadIdx.x; b < nblk; b += 32)
    for (int i = 0; i < 4; ++i) s[i] += partial[(long)b * 4 + i];
  for (int i = 0; i < 4; ++i) s[i] = warp_sum(s[i]);
  if (threadIdx.x != 0) return;
  if (maskout) {
    maskout[0] = (float)B;
    maskout[1] = (float)s[3];
  }
  if (mode == 0) return;
  const double Bg = denom ? (double)denom[0] : (double)B;
  const double Mg = denom ? (double)denom[1] : s[3];
  const double mse0 = s[0] / Bg, mse1 = s[1] / (Bg * O), mse2 = s[2] / (Mg * O);
  out[0] = (float)(p1 * mse0 + (1.0 - p1) * (p2 * mse1 + (1.0 - p2) * mse2));
  out[1] = (float)mse0;
}

// =============================================================================================
// RNNUqRangeEstimate head and loss (rnn_uq_range_estimate.py:104-108, model_utils/custom_layers.py:12-13,
// model_utils/losses.py:180-284).
// =============================================================================================
__device__ __forceinline__ float softplus_f(float a) { return fmaxf(a, 0.f) + log1pf(expf(-fabsf(a))); }

// var = max(softplus(a), 1e-6); in place when var == a
__global__ void softplus_floor_kernel(long n, const float* __restrict__ a, float* __restrict__ var) {
  const long i = (long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) var[i] = fmaxf(softplus_f(a[i]), 1e-6f);
}

int softplus_floor(cudaStream_t s, long n, const float* a, float* var) {
  softplus_floor_kernel<<<cdiv(n, 256), 256, 0, s>>>(n, a, var);
  LFMQ_LAUNCH_CHECK();
  return 0;
}

// One thread per [b,t] row.  Per element (losses.py:197-201,268-273): pm = p*m, vm = v*m, term = (pm-y)^2 * (1/vm) +
// log(vm) in fp32 exactly as written there -- a masked row gives 0*inf + log 0 = NaN, as in the reference; sums are
// carried in fp64.  pred == nullptr: only the two mask counts.  dpred != nullptr: gradients w.r.t. pred and w.r.t. the
// variance head's pre-activation `apre` (tf.maximum passes the gradient to softplus above the floor), using the counts
// of a previous pass.
__global__ void __launch_bounds__(256) uq_loss_rows_kernel(int B, int T, int O, const float* __restrict__ pred,
                                                           const float* __restrict__ var,
                                                           const float* __restrict__ apre,
                                                           const float* __restrict__ y,
                                                           const float* __restrict__ counts, int target_idx, float p1,
                                                           float p2, float* __restrict__ dpred,
                                                           float* __restrict__ da, double* __restrict__ partial) {
  double acc[4] = {0, 0, 0, 0};   // uq_0, uq_1, uq_2 numerators, mse_0 numerator
  double cnt[4] = {0, 0, 0, 0};   // unmasked rows, unmasked last-step rows
  float c_all = 0.f, c_last = 0.f, c_tar = 0.f;
  if (dpred) {
    const float ms_all = counts[0], ms_last = counts[1];
    c_all = (1.f - p1) * (1.f - p2) / (ms_all * (float)O);
    c_last = (1.f - p1) * p2 / (ms_last * (float)O);
    c_tar = p1 / ms_last;
  }
  const long rows = (long)B * T;
  for (long r = (long)blockIdx.x * blockDim.x + threadIdx.x; r < rows; r += (long)gridDim.x * blockDim.x) {
    const float* yr = y + r * O;
    bool any = false;
    for (int k = 0; k < O; ++k) any |= (yr[k] != 0.0f);
    const float m = any ? 1.f : 0.f;
    const bool last = ((int)(r % T) == T - 1);
    cnt[0] += m;
    if (last) cnt[1] += m;
    if (!pred) continue;
    for (int k = 0; k < O; ++k) {
      const float pm = pred[r * O + k] * m, vm = var[r * O + k] * m;
      const float d = pm - yr[k];
      const float diff = d * d;
      const float term = diff * (1.f / vm) + logf(vm);
      acc[2] += term;
      float coef = c_all;
      if (last) {
        acc[1] += term;
        coef += c_last;
        if (k == target_idx) { acc[0] += term; acc[3] += diff; coef += c_tar; }
      }
      if (dpred) {
        dpred[r * O + k] = coef * (2.f * d / vm) * m;
        const float dv = coef * (-diff / (vm * vm) + 1.f / vm) * m;
        const float a = apre[r * O + k];
        da[r * O + k] = dv * ((softplus_f(a) > 1e-6f) ? sigmoid_f(a) : 0.f);
      }
    }
  }
  block_reduce4(acc, partial + (long)blockIdx.x * 8);
  __syncthreads();
  block_reduce4(cnt, partial + (long)blockIdx.x * 8 + 4);
}

__global__ void uq_loss_final_kernel(int nblk, const double* __restrict__ partial, const float* __restrict__ counts_in,
                                     int B, int O, float p1, float p2, float* __restrict__ out_loss,
                                     float* __restrict__ out_uq0, float* __restrict__ out_mse0,
                                     float* __restrict__ counts_out) {
  double s[8] = {0, 0, 0, 0, 0, 0, 0, 0};
  for (int b = threadIdx.x; b < nblk; b += 32)
    for (int i = 0; i < 8; ++i) s[i] += partial[(long)b * 8 + i];
  for (int i = 0; i < 8; ++i) s[i] = warp_sum(s[i]);
  if (threadIdx.x != 0) return;
  if (counts_out) {
    counts_out[0] = (float)s[4];
    counts_out[1] = (float)s[5];
  }
  if (!out_loss) return;
  const double ms_all = counts_in ? (double)counts_in[0] : s[4];
  const double ms_last = counts_in ? (double)counts_in[1] : s[5];
  const double uq0 = s[0] / ms_last, uq1 = s[1] / (ms_last * O), uq2 = s[2] / (ms_all * O);
  *out_loss = (float)(p1 * uq0 + (1.0 - p1) * (p2 * uq1 + (1.0 - p2) * uq2));
  *out_uq0 = (float)uq0;
  *out_mse0 = (float)(s[3] / (double)B);
}

// pred == nullptr: counts only -> counts_out.  Otherwise the three scalars; with dpred also the gradients (counts_in
// from a counts-only pass is then required).
int uq_loss_grad(cudaStream_t s, int B, int T, int O, const float* pred, const float* var, const float* apre,
                 const float* y, const float* counts_in, int target_idx, float p1, float p2, float* dpred, float* da,
                 float* out_loss, float* out_uq0, float* out_mse0, float* counts_out, float* scratch) {
  double* partial = reinterpret_cast<double*>(scratch);
  uq_loss_rows_kernel<<<LOSS_BLOCKS, 256, 0, s>>>(B, T, O, pred, var, apre, y, counts_in, target_idx, p1, p2, dpred, da,
                                                  partial);
  LFMQ_LAUNCH_CHECK();
  uq_loss_final_kernel<<<1, 32, 0, s>>>(LOSS_BLOCKS, partial, counts_in, B, O, p1, p2, out_loss, out_uq0, out_mse0,
                                        counts_out);
  LFMQ_LAUNCH_CHECK();
  return 0;
}

// mask count (losses.py:72-73,132): one thread per [b,t] row, warp ballot, one integer atomic per warp
// (integer adds commute: the count is exact and deterministic).  The last block to finish (ticket) writes
// {B, count} and resets both counters, so the whole count is one launch and needs no memset.
__global__ void __launch_bounds__(256) mask_rows_kernel(long rows, int O, int B, const float* __restrict__ y,
                                                        unsigned int* __restrict__ tickets,
                                                        float* __restrict__ out2) {
  pdl_sync();
  const long r = (long)blockIdx.x * blockDim.x + threadIdx.x;
  bool any = false;
  if (r < rows) {
    const float* yr = y + r * O;
    if ((O & 3) == 0) {
      for (int k = 0; k < O; k += 4) {
        const float4 v = *reinterpret_cast<const float4*>(yr + k);
        any |= (v.x != 0.f) | (v.y != 0.f) | (v.z != 0.f) | (v.w != 0.f);
      }
    } else {
      for (int k = 0; k < O; ++k) any |= (yr[k] != 0.f);
    }
  }
  const unsigned int bal = __ballot_sync(0xffffffffu, any);
  if ((threadIdx.x & 31) == 0 && bal) atomicAdd(&tickets[0], (unsigned int)__popc(bal));
  __syncthreads();
  if (threadIdx.x == 0) {
    __threadfence();
    if (atomicAdd(&tickets[1], 1u) == gridDim.x - 1) {
      __threadfence();
      const unsigned int c = atomicExch(&tickets[0], 0u);
      out2[0] = (float)B;
      out2[1] = (float)c;
      tickets[1] = 0u;
    }
  }
}

int mask_count(cudaStream_t s, int B, int T, int O, const float* y, float* out2, unsigned int* tickets) {
  const long rows = (long)B * T;
  if (int rc = launch_pdl(mask_rows_kernel, dim3(cdiv(rows, 256)), dim3(256), 0, s, 1, true, rows, O, B, y, tickets, out2)) return rc;
  return 0;
}

int loss_grad(cudaStream_t s, int B, int T, int O, const float* pred, const float* y, const float* denom,
              int target_idx, float p1, float p2, float* dpred, float* out2, float* maskout2, float* scratch) {
  double* partial = reinterpret_cast<double*>(scratch);
  loss_rows_kernel<<<LOSS_BLOCKS, 256, 0, s>>>(B, T, O, pred, y, denom, target_idx, p1, p2, dpred, partial);
  LFMQ_LAUNCH_CHECK();
  loss_final_kernel<<<1, 32, 0, s>>>(LOSS_BLOCKS, partial, denom, B, O, p1, p2, 1, out2, maskout2);
  LFMQ_LAUNCH_CHECK();
  return 0;
}

// =============================================================================================
// clip_by_global_norm + optimizer + MaxNorm (train.py:195-198, model_utils/optimizers.py:21-27,
// rnn_point_estimate.py:85; SURVEY App. A.5).
// =============================================================================================
// Sum of squares in fp64 partials; the last block to finish (ticket) adds the partials in block order -- the result
// does not depend on which block that is -- and writes {norm, clip scale}.  One launch, self-resetting ticket.
__global__ void __launch_bounds__(256) sumsq_norm_kernel(long n, const float* __restrict__ g,
                                                         double* __restrict__ partial, float clip,
                                                         float* __restrict__ scalars,
                                                         unsigned int* __restrict__ ticket) {
  pdl_sync();
  double acc[4] = {0, 0, 0, 0};
  for (long i = (long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long)gridDim.x * blockDim.x) {
    const double v = g[i];
    acc[0] += v * v;
  }
  block_reduce4(acc, partial + (long)blockIdx.x * 4);
  __shared__ bool last;
  __syncthreads();                     // block_reduce4's writers (threads 0-3) are done
  if (threadIdx.x == 0) {
    __threadfence();
    last = atomicAdd(ticket, 1u) == gridDim.x - 1;
  }
  __syncthreads();
  if (!last || threadIdx.x >= 32) return;
  __threadfence();
  double s = 0;
  for (int b = threadIdx.x; b < (int)gridDim.x; b += 32) s += __ldcg(partial + (long)b * 4);
  s = warp_sum(s);
  if (threadIdx.x != 0) return;
  const float gn = (float)sqrt(s);
  scalars[0] = gn;
  scalars[1] = (clip > 0.f) ? clip / fmaxf(gn, clip) : 1.0f;
  *ticket = 0u;
}

int grad_norm_scale(cudaStream_t s, long n, const float* g, float clip, float* scalars, float* scratch,
                    unsigned int* ticket) {
  double* partial = reinterpret_cast<double*>(scratch);
  const int nblk = (int)min((long)device_sm_count(), max((long)1, n / 2048));
  if (int rc = launch_pdl(sumsq_norm_kernel, dim3(nblk), dim3(256), 0, s, 1, true, n, g, partial, clip, scalars, ticket)) return rc;
  return 0;
}

__global__ void opt_update_kernel(int opt, long n, float* __restrict__ p, const float* __restrict__ g,
                                  float* __restrict__ s0, float* __restrict__ s1,
                                  const float* __restrict__ scalars, float lr, float momentum) {
  pdl_sync();
  const long i = (long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const float gr = g[i] * scalars[1];
  float w = p[i];
  if (opt == 0) {            // Adadelta rho=.95 eps=1e-7
    const float rho = 0.95f, eps = 1e-7f;
    const float a = rho * s0[i] + (1.f - rho) * gr * gr;
    const float upd = sqrtf(s1[i] + eps) / sqrtf(a + eps) * gr;
    s0[i] = a;
    s1[i] = rho * s1[i] + (1.f - rho) * upd * upd;
    w -= lr * upd;
  } else if (opt == 1) {     // Adam, lr already bias-corrected on the host
    const float b1 = 0.9f, b2 = 0.999f, eps = 1e-7f;
    const float m = b1 * s0[i] + (1.f - b1) * gr;
    const float v = b2 * s1[i] + (1.f - b2) * gr * gr;
    s0[i] = m;
    s1[i] = v;
    w -= lr * m / (sqrtf(v) + eps);
  } else if (opt == 2) {     // RMSprop rho=.9 eps=1e-7
    const float rho = 0.9f, eps = 1e-7f;
    const float v = rho * s0[i] + (1.f - rho) * gr * gr;
    s0[i] = v;
    w -= lr * gr / (sqrtf(v) + eps);
  } else {                   // SGD (+ momentum)
    if (momentum > 0.f) {
      const float m = momentum * s0[i] - lr * gr;
      s0[i] = m;
      w += m;
    } else {
      w -= lr * gr;
    }
  }
  p[i] = w;
}

int opt_update(cudaStream_t s, int opt, long n, float* p, const float* g, float* slot0, float* slot1,
               const float* scalars, float lr, float, float, float momentum) {
  if (int rc = launch_pdl(opt_update_kernel, dim3(cdiv(n, 256)), dim3(256), 0, s, 1, true, opt, n, p, g, slot0, slot1, scalars, lr, momentum)) return rc;
  return 0;
}

// keras.constraints.MaxNorm(max_value, axis=0) on W[I,N]: one warp per column (lanes stride the rows; a thread per
// column left 2048 threads walking 512 dependent rows each).
__global__ void maxnorm_cols_kernel(int I, int N, float* __restrict__ W, float max_norm) {
  pdl_sync();
  const int n = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (n >= N) return;
  float ss = 0.f;
  for (int i = lane; i < I; i += 32) {
    const float v = W[(long)i * N + n];
    ss = fmaf(v, v, ss);
  }
  ss = warp_sum(ss);
  const float nr = sqrtf(ss);
  const float f = fminf(fmaxf(nr, 0.f), max_norm) / (1e-7f + nr);
  for (int i = lane; i < I; i += 32) W[(long)i * N + n] *= f;
}

int maxnorm_cols(cudaStream_t s, int I, int N, float* W, float max_norm) {
  if (int rc = launch_pdl(maxnorm_cols_kernel, dim3(cdiv((long)N * 32, 256)), dim3(256), 0, s, 1, true, I, N, W, max_norm)) return rc;
  return 0;
}

// =============================================================================================
// Sliding-window batcher (data_processing.py:307-368, 370-449, 600-609; SURVEY App. A.6).
// One CTA per window; fp64 arithmetic then cast to fp32, as the reference.
// =============================================================================================
__device__ __forceinline__ double squash(double v) {
  // np.sign(v) * np.log1p(np.abs(v)); NaN propagates
  const double sg = (v > 0.0) ? 1.0 : ((v < 0.0) ? -1.0 : ((v == 0.0) ? 0.0 : v));
  return sg * log1p(fabs(v));
}

__global__ void __launch_bounds__(128) gather_batch_kernel(GatherArgs a) {
  const int b = blockIdx.x;
  const int is = a.inp_idx[b * 3 + 0], ipad = a.inp_idx[b * 3 + 2];
  const int ts = a.tar_idx[b * 3 + 0], te = a.tar_idx[b * 3 + 1], tpad = a.tar_idx[b * 3 + 2];
  double norm = 1.0;
  if (a.seq_norm_col >= 0) {
    // data_processing.py:393-396: max(seq[-1, idx], 10) with Python max() NaN semantics
    const long rl = (long)is + (long)(a.T - 1 - ipad) * a.stride;
    const double v = a.table[rl * a.n_cols + a.seq_norm_col];
    norm = (10.0 > v) ? 10.0 : v;
  }
  if (threadIdx.x == 0) a.seq_norm[b] = norm;
  const double qnan = __longlong_as_double(0x7ff8000000000000LL);
  for (int e = threadIdx.x; e < a.T * a.F; e += blockDim.x) {
    const int t = e / a.F, f = e % a.F;
    double v = 0.0;
    if (t >= ipad) v = a.table[((long)is + (long)(t - ipad) * a.stride) * a.n_cols + a.inp_cols[f]];
    if (f < a.O) {
      v /= norm;
      if (a.log_squasher) v = squash(v);
    }
    if (a.scale_flag[f]) v = (v - a.center[f]) / a.scale[f];
    if (a.aux_masking && a.aux_flag[f] && t < a.T - 1) v = 0.0;
    a.x[((long)b * a.T + t) * a.F + f] = (float)v;
  }
  for (int e = threadIdx.x; e < a.T * a.O; e += blockDim.x) {
    const int t = e / a.O, k = e % a.O;
    double v = 0.0;
    if (t >= tpad) {
      const long r = (long)ts + (long)(t - tpad) * a.stride;
      v = (r <= te && r < a.n_rows) ? a.table[r * a.n_cols + a.fin_cols[k]] : qnan;  // :427-435
    }
    v /= norm;
    if (a.log_squasher) v = squash(v);
    v = (v - a.center[k]) / a.scale[k];
    a.y[((long)b * a.T + t) * a.O + k] = (float)v;
  }
}

// Vectorised variant (F % 4 == 0, O % 4 == 0, F <= 256): one CTA per window, the per-column metadata (column ids,
// centre / scale, flags) staged in shared memory once, every thread item = 4 consecutive columns of one time step:
// two 128-bit fp64 loads when the 4 table columns are adjacent and 16-byte aligned (the usual case: the financial and
// aux fields are column ranges of the data file), one 128-bit fp32 store.  Same fp64 arithmetic, same results.
constexpr int GV_MAXF = 256;

__device__ __forceinline__ void gather_load4(const double* __restrict__ row, const int* cols, double v[4]) {
  const int c0 = cols[0];
  const bool adj = (cols[1] == c0 + 1) && (cols[2] == c0 + 2) && (cols[3] == c0 + 3);
  const double* p = row + c0;
  if (adj && ((reinterpret_cast<uintptr_t>(p) & 15) == 0)) {
    const double2 a = __ldg(reinterpret_cast<const double2*>(p));
    const double2 b = __ldg(reinterpret_cast<const double2*>(p) + 1);
    v[0] = a.x; v[1] = a.y; v[2] = b.x; v[3] = b.y;
  } else {
#pragma unroll
    for (int i = 0; i < 4; ++i) v[i] = __ldg(row + cols[i]);
  }
}

__global__ void __launch_bounds__(128) gather_batch_vec_kernel(GatherArgs a) {
  __shared__ int icol_s[GV_MAXF], fcol_s[GV_MAXF];
  __shared__ double cen_s[GV_MAXF], isc_s[GV_MAXF];      // centre, scale of column f (targets use the first O entries)
  __shared__ unsigned char sfl_s[GV_MAXF], afl_s[GV_MAXF];
  const int b = blockIdx.x;
  for (int f = threadIdx.x; f < a.F; f += blockDim.x) {
    icol_s[f] = a.inp_cols[f];
    cen_s[f] = a.center[f];
    isc_s[f] = a.scale[f];
    sfl_s[f] = a.scale_flag[f];
    afl_s[f] = a.aux_flag[f];
    if (f < a.O) fcol_s[f] = a.fin_cols[f];
  }
  const int is = a.inp_idx[b * 3 + 0], ipad = a.inp_idx[b * 3 + 2];
  const int ts = a.tar_idx[b * 3 + 0], te = a.tar_idx[b * 3 + 1], tpad = a.tar_idx[b * 3 + 2];
  double norm = 1.0;
  if (a.seq_norm_col >= 0) {
    const long rl = (long)is + (long)(a.T - 1 - ipad) * a.stride;
    const double v = __ldg(a.table + rl * a.n_cols + a.seq_norm_col);
    norm = (10.0 > v) ? 10.0 : v;
  }
  if (threadIdx.x == 0) a.seq_norm[b] = norm;
  __syncthreads();
  const double qnan = __longlong_as_double(0x7ff8000000000000LL);
  const int F4 = a.F >> 2, O4 = a.O >> 2;
  for (int e = threadIdx.x; e < a.T * F4; e += blockDim.x) {
    const int t = e / F4, f = (e - t * F4) << 2;
    double v[4] = {0.0, 0.0, 0.0, 0.0};
    if (t >= ipad) gather_load4(a.table + ((long)is + (long)(t - ipad) * a.stride) * a.n_cols, icol_s + f, v);
    float o[4];
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      double w = v[i];
      if (f + i < a.O) {
        w /= norm;
        if (a.log_squasher) w = squash(w);
      }
      if (sfl_s[f + i]) w = (w - cen_s[f + i]) / isc_s[f + i];
      if (a.aux_masking && afl_s[f + i] && t < a.T - 1) w = 0.0;
      o[i] = (float)w;
    }
    *reinterpret_cast<float4*>(a.x + ((long)b * a.T + t) * a.F + f) = make_float4(o[0], o[1], o[2], o[3]);
  }
  for (int e = threadIdx.x; e < a.T * O4; e += blockDim.x) {
    const int t = e / O4, k = (e - t * O4) << 2;
    double v[4] = {0.0, 0.0, 0.0, 0.0};
    if (t >= tpad) {
      const long r = (long)ts + (long)(t - tpad) * a.stride;
      if (r <= te && r < a.n_rows) gather_load4(a.table + r * a.n_cols, fcol_s + k, v);
      else v[0] = v[1] = v[2] = v[3] = qnan;                              // :427-435
    }
    float o[4];
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      double w = v[i] / norm;
      if (a.log_squasher) w = squash(w);
      w = (w - cen_s[k + i]) / isc_s[k + i];
      o[i] = (float)w;
    }
    *reinterpret_cast<float4*>(a.y + ((long)b * a.T + t) * a.O + k) = make_float4(o[0], o[1], o[2], o[3]);
  }
}

int gather_batch(cudaStream_t s, const GatherArgs& a) {
  if (a.B <= 0) return 0;
  const bool vec = (a.F % 4 == 0) && (a.O % 4 == 0) && a.F <= GV_MAXF &&
                   ((reinterpret_cast<uintptr_t>(a.x) | reinterpret_cast<uintptr_t>(a.y)) & 15) == 0;
  if (vec)
    gather_batch_vec_kernel<<<a.B, 128, 0, s>>>(a);
  else
    gather_batch_kernel<<<a.B, 128, 0, s>>>(a);
  LFMQ_LAUNCH_CHECK();
  return 0;
}

// Train._unscale_preds (train.py:420-432): affine un-scaling + reverse log-squash, fp64 then cast.
__global__ void unscale_kernel(long n, int O, const float* __restrict__ in, float* __restrict__ out,
                               const double* __restrict__ scale, const double* __restrict__ center, int log_squasher) {
  const long i = (long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const int k = (int)(i % O);
  double v = (double)in[i] * scale[k] + center[k];
  if (log_squasher) {
    const double sg = (v > 0.0) ? 1.0 : ((v < 0.0) ? -1.0 : ((v == 0.0) ? 0.0 : v));
    v = sg * expm1(fabs(v));
  }
  out[i] = (float)v;
}

int unscale(cudaStream_t s, const float* in, float* out, long n_rows, int O, const double* scale, const double* center,
            int log_squasher) {
  const long n = n_rows * O;
  if (n <= 0) return 0;
  unscale_kernel<<<cdiv(n, 256), 256, 0, s>>>(n, O, in, out, scale, center, log_squasher);
  LFMQ_LAUNCH_CHECK();
  return 0;
}

}  // namespace lfmq
