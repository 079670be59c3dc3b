// LFMQ_PREC_BF16: the gate GEMMs on Hopper tensor cores (wgmma: bf16 operands from shared memory, fp32 accumulation
// in the registers of the issuing warpgroup, fp32 cell state in registers, bf16 when saved), everything else as fused
// HBM-streaming kernels.  sm_90a.
//
// Data layout in HBM (all carved from the caller's workspace, see tc_layout):
//   xh    bf16 [maxB][T+1][384]   row (b,t): cols 0..255 = h_{t-1} (zero at t=0), 256..287 = x_t, 288 = 1.0 (t<T),
//                                 rest 0.  One buffer serves: the A operand of the forward recurrence (K-major
//                                 tiles via TMA), the head (h_t = row t+1) and the weight-gradient GEMM (MN-major).
//   gates bf16 [T][tiles][8 blocks of 32 units][4 row quadrants][8 pieces = gate*2+half][32 rows][16]   post-activation
//                                 i|f|g|o saved for BPTT, SoA at 32-byte granularity (row-major within a piece)
//   cst   bf16 [T][tiles][8][4][2 pieces][32][16]   cell states (the recurrence itself keeps them in fp32 registers)
//   dz    bf16 [maxB][T+1][4H]    gate pre-activation gradients (row T stays zero); columns in the order the
//                                 backward kernel stages them as its A operand, [16-unit block][gate][16], so that a
//                                 chunk goes out with one TMA store; only the weight-gradient GEMM reads it
//   dpb   bf16 [T][tiles][128][32]  dLoss/dpred tiles (cols >= 16 zero): written by the tensor-core head as it stages
//                                 them, expanded to dLoss/dh by the backward kernel's own MMAs (no dropout)
//   dhout bf16 [T][tiles][4 ranks][4 row quadrants][4 chunks][32 rows][16]   dropout > 0 only: dLoss/dh from the SIMT
//                                 head (after BN/dropout backward)
//
// Forward recurrence = ONE persistent kernel (lstm_fwd_tc_kernel): clusters of 4 CTAs, one 128-row batch tile per
// cluster, all clusters co-resident.  CTA r keeps the weight slice of hidden units [64r, 64r+64) (all four gates,
// 256 gate columns) resident in shared memory for the whole unroll.  h_t is exchanged through global memory (it is
// an output anyway) and comes back as the next step's A operand via TMA multicast.  See DESIGN.md section 5.
#include "lstm_tc.h"

#include <cuda.h>
#include <cuda_bf16.h>
#include <stdlib.h>

#include "kernels.h"
#include "sm90.cuh"

namespace lfmq {

using namespace sm90;

namespace {

constexpr int TC_H = 256;          // hidden units (bf16 path is specialised for H = 256)
constexpr int TC_NC = 4;           // CTAs per forward cluster
constexpr int TC_HS = 64;          // hidden units per forward CTA
constexpr int TC_NSL = 256;        // gate columns per forward CTA
constexpr int TC_XH_LD = 384;      // elements per xh row
constexpr int TC_XOFF = 256;       // first x column inside an xh row
constexpr int TC_ONE = 288;        // the constant-one column (db falls out of the weight-gradient GEMM)
constexpr int TC_OPAD = 16;        // head handles n_outputs <= 16

}  // namespace

struct TcImpl {
  bool enabled = false;
  int maxB = 0, T = 0, I = 0, O = 0;
  float eps = 1e-3f;
  // parameter offsets in the flat fp32 vector (L = 1)
  int64_t oW, oU, ob, ogamma, obeta, oWo, obo, omean, ovar;
  // workspace
  bool train = false;                          // training handle: saved state and the backward recurrence exist
  __nv_bfloat16 *xh, *gates, *dz, *dhout, *Up, *Wp, *Ubk;
  __nv_bfloat16* cst;
  float *biasp, *head_part, *head_wpart, *dpred, *wg_part;
  size_t head_part_elems, wg_part_elems;
  CUtensorMap tm_h, tm_x, tm_u, tm_w;          // forward
  CUtensorMap tm_h128, tm_wot;                 // head: 128-row h tiles, folded head weights
  __nv_bfloat16* WoTp;
  __nv_bfloat16* WoSp;                         // [256][32]  Wo[j][k] * gamma_j * inv_j (k < 16), zero padded
  __nv_bfloat16* dpb;                          // [T][tiles][128][32] bf16 dLoss/dpred tiles (cols >= 16 zero)
  CUtensorMap tm_wos, tm_dpb;
  float* bop;
  CUtensorMap tm_ubk;                          // backward recurrence
  CUtensorMap tm_xh_mn, tm_dz_mn;              // weight gradient (MN-major)
  int max_clusters = 0, bwd_max_clusters = 0;
  bool bwd_ready = false;
  int head_ctas = 0, head_wctas = 0;
  int n_sms = 0;
};

// =============================================================================================
// Small packing / cast kernels
// =============================================================================================
// x f32 [B,T,F] -> xh[b][t][256 .. 256+F), plus the constant-one column.  One 16-byte chunk per thread.
__global__ void xh_fill_x_kernel(int B, int T, int F, const float* __restrict__ x, __nv_bfloat16* __restrict__ xh) {
  pdl_sync();
  const long idx = (long)blockIdx.x * blockDim.x + threadIdx.x;   // (row, chunk) with 5 chunks of 8 columns per row
  if (idx >= (long)B * T * 5) return;
  const long row = idx / 5;
  const int c = (int)(idx % 5);
  const long b = row / T;
  const int t = (int)(row % T);
  float v[8];
#pragma unroll
  for (int e = 0; e < 8; ++e) {
    const int f = c * 8 + e;
    v[e] = (f < F) ? x[row * F + f] : ((f == TC_ONE - TC_XOFF) ? 1.0f : 0.f);
  }
  uint4 o;
  o.x = pack_bf16x2(v[0], v[1]);
  o.y = pack_bf16x2(v[2], v[3]);
  o.z = pack_bf16x2(v[4], v[5]);
  o.w = pack_bf16x2(v[6], v[7]);
  *reinterpret_cast<uint4*>(xh + (b * (T + 1) + t) * TC_XH_LD + TC_XOFF + c * 8) = o;
}

// Weight slices in the order the forward kernel consumes them.  Gate g of hidden unit 64r + 16c + jj is row
// n = 64c + 16g + jj of slice r (four 16-unit chunks of 64 gate columns each: the MMAs are issued and committed two
// chunks at a time, so the epilogue of chunks 0-1 runs under the MMAs of chunks 2-3); the three sigmoid gates are pre-scaled by 0.5
// (sigmoid(z) = 0.5*tanh(z/2) + 0.5).
__device__ __forceinline__ void pack_weights_body(int bid, int I, const float* __restrict__ W, const float* __restrict__ U,
                                    const float* __restrict__ bias, __nv_bfloat16* __restrict__ Up,
                                    __nv_bfloat16* __restrict__ Wp, float* __restrict__ biasp) {
  const int H = TC_H;
  const long idx = (long)bid * blockDim.x + threadIdx.x;
  if (idx < (long)4 * H * H) {          // Up: [4][256][256]
    const int k = (int)(idx % H);
    const int n = (int)((idx / H) % TC_NSL);
    const int r = (int)(idx / ((long)H * TC_NSL));
    const int g = (n % 64) / 16, j = (n / 64) * 16 + n % 16;
    const float sc = (g == 2) ? 1.0f : 0.5f;
    Up[idx] = __float2bfloat16(sc * U[(long)k * 4 * H + g * H + r * TC_HS + j]);
  }
  if (idx < (long)4 * H * 32) {         // Wp: [4][256][32]
    const int k = (int)(idx % 32);
    const int n = (int)((idx / 32) % TC_NSL);
    const int r = (int)(idx / (32 * TC_NSL));
    const int g = (n % 64) / 16, j = (n / 64) * 16 + n % 16;
    const float sc = (g == 2) ? 1.0f : 0.5f;
    Wp[idx] = __float2bfloat16(k < I ? sc * W[(long)k * 4 * H + g * H + r * TC_HS + j] : 0.f);
  }
  if (idx < 4 * H) {                    // biasp: [4][256]
    const int n = (int)(idx % TC_NSL), r = (int)(idx / TC_NSL);
    const int g = (n % 64) / 16, j = (n / 64) * 16 + n % 16;
    biasp[idx] = ((g == 2) ? 1.0f : 0.5f) * bias[g * H + r * TC_HS + j];
  }
}

// =============================================================================================
// Persistent forward recurrence
// =============================================================================================
struct FwdParams {
  int B, T, n_iters, n_clusters, n_tiles, k16_x, n_tiles_cap;
  __nv_bfloat16* xh;
  __nv_bfloat16* gates;   // null: do not save
  __nv_bfloat16* cst;     // null: do not save
  const float* biasp;
};

// Warps 0-7: two consumer warpgroups (rows 0-63 / 64-127 of the tile; each issues its own wgmma and runs the cell
// update on its accumulator fragment); warpgroup 2: warp 8 = TMA producer.  setmaxnreg moves the registers of the
// producer warpgroup to the consumers (128 accumulators + 32 cell states per thread).
constexpr int FWD_THREADS = 3 * 128;
constexpr int FWD_PRODUCER_WARP = 8;
constexpr uint32_t SM_U = 0;                 // 4 k-blocks x [256 x 128 B]
constexpr uint32_t SM_W = 131072;            // [256 x 64 B]
constexpr uint32_t SM_H0 = 147456;           // 4 k-blocks x [128 x 128 B]
constexpr uint32_t SM_X0 = 212992;           // [128 x 64 B]
constexpr uint32_t SM_BIAS = 221184;
constexpr uint32_t SM_BARS = 222208;
constexpr uint32_t FWD_SMEM = SM_BARS + 256 + 1024;   // + alignment slack

struct FwdBars {
  uint64_t w_full, x_full, x_empty, h_full, h_written;
};

// Post-activation gates i|f|g|o of units jj, jj + 1 (row half h, pair q) from a 64-column chunk of the accumulator:
// gate g of unit jj + e is fragment register 4 (2 g + q) + 2 h + e.  The sigmoid gates come pre-scaled by 1/2.
__device__ __forceinline__ void fwd_gates(const float* a, const float* bs, int h, int q, int jj, float (&gv)[4][2]) {
#pragma unroll
  for (int e = 0; e < 2; ++e) {
    const int ri = 2 * h + e;
    gv[0][e] = fmaf(0.5f, tanh_approx(a[4 * (0 + q) + ri] + bs[jj + e]), 0.5f);
    gv[1][e] = fmaf(0.5f, tanh_approx(a[4 * (2 + q) + ri] + bs[16 + jj + e]), 0.5f);
    gv[2][e] = tanh_approx(a[4 * (4 + q) + ri] + bs[32 + jj + e]);
    gv[3][e] = fmaf(0.5f, tanh_approx(a[4 * (6 + q) + ri] + bs[48 + jj + e]), 0.5f);
  }
}

// SAVE: training (gates / cell states kept for BPTT).  A template parameter so that the predict kernel carries none of
// the saved-state logic.
template <bool SAVE>
__global__ void __launch_bounds__(FWD_THREADS, 1)
    lstm_fwd_tc_kernel(FwdParams p, const __grid_constant__ CUtensorMap tm_h, const __grid_constant__ CUtensorMap tm_x,
                       const __grid_constant__ CUtensorMap tm_u, const __grid_constant__ CUtensorMap tm_w) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  FwdBars* bars = reinterpret_cast<FwdBars*>(smem + SM_BARS);
  float* bias_s = reinterpret_cast<float*>(smem + SM_BIAS);
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const uint32_t rank = cluster_ctarank();
  const int cid = blockIdx.x / TC_NC;

  if (tid == 0) {
    mbar_init(&bars->w_full, 1);
    mbar_init(&bars->x_full, 1);
    mbar_init(&bars->x_empty, 8);           // one arrive per consumer warp
    mbar_init(&bars->h_full, 1);
    mbar_init(&bars->h_written, TC_NC);
    fence_mbar_init();
  }
  if (tid < TC_NSL) bias_s[tid] = p.biasp[rank * TC_NSL + tid];
  __syncthreads();
  cluster_sync_all();          // peers' barriers are initialised before anyone multicasts / arrives remotely
  const int T = p.T;
  // Programmatic dependent launch: everything above and the weight slice (packed two kernels ago) do not depend on the
  // preceding kernel (xh_fill_x); the 144 KB weight load overlaps its tail.
  if (!(warp == FWD_PRODUCER_WARP && lane == 0)) pdl_sync();

  if (warp >= FWD_PRODUCER_WARP) {
    setmaxnreg_dec<40>();
    // ===================== TMA producer =====================
    if (warp == FWD_PRODUCER_WARP && lane == 0) {
      mbar_arrive_expect_tx(&bars->w_full, 131072 + 16384);
      for (int kb = 0; kb < 4; ++kb) tma_load_2d(smem + SM_U + kb * 32768, &tm_u, &bars->w_full, kb * 64, rank * TC_NSL);
      tma_load_2d(smem + SM_W, &tm_w, &bars->w_full, 0, rank * TC_NSL);
      pdl_sync();
      uint8_t* hbuf = smem + SM_H0;
      uint8_t* xbuf = smem + SM_X0;
      uint32_t n_hw = 0, n_xe = 0;
      for (int it = 0; it < p.n_iters; ++it) {
        if (it * p.n_clusters + cid >= p.n_tiles) break;   // clusters without a tile in the last round
        const int b0 = (it * p.n_clusters + cid) * 128;
        for (int t = 0; t < T; ++t) {
          if (it > 0 || t > 0) mbar_wait(&bars->x_empty, (n_xe++) & 1);
          mbar_arrive_expect_tx(&bars->x_full, 8192);
          tma_load_2d(xbuf, &tm_x, &bars->x_full, t * TC_XH_LD + TC_XOFF, b0);
          if (t >= 1) {
            mbar_wait_cluster(&bars->h_written, (n_hw++) & 1);   // all 4 slices of h_{t-1} are in global memory
            fence_proxy_async_global();
            mbar_arrive_expect_tx(&bars->h_full, 65536);
            for (int kb = 0; kb < 4; ++kb)
              tma_load_2d_mcast(hbuf + kb * 16384 + rank * 4096, &tm_h, &bars->h_full, t * TC_XH_LD + kb * 64,
                                b0 + 32 * (int)rank, 0xF);
          }
        }
        mbar_wait_cluster(&bars->h_written, (n_hw++) & 1);       // phase of step T-1 (keeps parities aligned)
      }
    }
  } else {
    setmaxnreg_inc<232>();
    // ===================== consumers: gate GEMMs, gates, cell update, h exchange =====================
    // Accumulator of warpgroup wg: rows 64 wg .. 64 wg + 63, four 64-column chunks (one per 16 hidden units).  In chunk
    // c the thread holds, for rows r0 and r0 + 8, the four gates of units jj = 8 p + 2 cq + e (p, e in {0, 1}):
    // gate g of unit jj is fragment register 4 (2 g + p) + 2 h + e.  The cell state of those 2 x 16 values stays in
    // fp32 registers for the whole unroll.
    const int wg = warp >> 2, w = warp & 3, cq = lane & 3;
    const int r0 = 64 * wg + 16 * w + (lane >> 2);
    mbar_wait(&bars->w_full, 0);
    uint32_t n_xf = 0, n_hf = 0;
    float acc[2][64];                       // [half g]: chunks 2 g (registers 0-31) and 2 g + 1 (32-63)
    float cstate[4][2][2][2];               // [chunk][row half h][pair p][e]
    for (int it = 0; it < p.n_iters; ++it) {
      const int tile_c = it * p.n_clusters + cid;
      if (tile_c >= p.n_tiles) break;
#pragma unroll
      for (int c = 0; c < 4; ++c)
#pragma unroll
        for (int h = 0; h < 2; ++h)
#pragma unroll
          for (int q = 0; q < 2; ++q) cstate[c][h][q][0] = cstate[c][h][q][1] = 0.f;
      for (int t = 0; t < T; ++t) {
        // Two 128-column halves (chunks 2 g, 2 g + 1: an m64n128 fragment is the two m64n64 fragments side by side), each
        // its own commit group for the h part: the cell update of chunks 0-1 overlaps the MMAs of chunks 2-3.  Against
        // one group per 64-column chunk, each k-step re-reads the h tile's A operand from shared memory half as often.
        // The x part of both halves goes first: it does not wait for h.
        mbar_wait(&bars->x_full, (n_xf++) & 1);
        wgmma_fence();
#pragma unroll
        for (int g = 0; g < 2; ++g)
          for (int k16 = 0; k16 < p.k16_x; ++k16) {
            const uint64_t da = make_smem_desc(smem_u32(smem + SM_X0 + wg * 4096) + k16 * 32, 0, 512, LAYOUT_SW64);
            const uint64_t db = make_smem_desc(smem_u32(smem + SM_W + g * 8192) + k16 * 32, 0, 512, LAYOUT_SW64);
            wgmma_m64n128k16<0, 0>(acc[g], da, db, k16 > 0);
          }
        wgmma_commit();
        if (t > 0) {
          mbar_wait(&bars->h_full, (n_hf++) & 1);
#pragma unroll
          for (int g = 0; g < 2; ++g) {
#pragma unroll
            for (int kb = 0; kb < 4; ++kb)
#pragma unroll
              for (int k16 = 0; k16 < 4; ++k16) {
                const uint64_t da = make_smem_desc(smem_u32(smem + SM_H0 + kb * 16384 + wg * 8192) + k16 * 32, 0, 1024,
                                                   LAYOUT_SW128);
                const uint64_t db = make_smem_desc(smem_u32(smem + SM_U + kb * 32768 + g * 16384) + k16 * 32, 0, 1024,
                                                   LAYOUT_SW128);
                wgmma_m64n128k16<0, 0>(acc[g], da, db, 1);
              }
            wgmma_commit();
          }
          wgmma_wait<2>();
        } else {
          wgmma_wait<0>();
        }
        if (lane == 0) mbar_arrive(&bars->x_empty);      // the x tile has been read
#pragma unroll
        for (int c = 0; c < 4; ++c) {
          // Unconditional although nothing is in flight at t = 0: behind a branch on t, ptxas cannot follow the commit
          // groups and serialises every wgmma of the kernel (C7514).
          if (c == 0) wgmma_wait<1>();
          if (c == 2) wgmma_wait<0>();
          if ((c & 1) == 0) fence_regs(acc[c >> 1]);
          const float* ac = acc[c >> 1] + 32 * (c & 1);
          const float* bs = bias_s + c * 64;
#pragma unroll
          for (int h = 0; h < 2; ++h) {
            const int m = r0 + 8 * h;               // row of the 128-row tile
            const long b = (long)tile_c * 128 + m;
#pragma unroll
            for (int q = 0; q < 2; ++q) {
              const int jj = 8 * q + 2 * cq;          // first of the two units of this pair
              float gv[4][2], hv[2];
              fwd_gates(ac, bs, h, q, jj, gv);
#pragma unroll
              for (int e = 0; e < 2; ++e) {
                const float cc = fmaf(gv[1][e], cstate[c][h][q][e], gv[0][e] * gv[2][e]);
                cstate[c][h][q][e] = cc;
                hv[e] = gv[3][e] * tanh_approx(cc);
              }
              if (b < p.B)
                *reinterpret_cast<uint32_t*>(p.xh + (b * (T + 1) + (t + 1)) * TC_XH_LD + rank * TC_HS + c * 16 + jj) =
                    pack_bf16x2(hv[0], hv[1]);
            }
          }
        }
        // Publish this CTA's h slice: barrier over the 256 consumer threads, then 4 lanes of warp 0 arrive
        // (release.cluster, cumulative over the barrier) on the 4 CTAs' h_written barriers in parallel.  Readers acquire
        // at cluster scope and cross into the async proxy before their TMA loads.  All MMAs of the step are complete
        // here, so the h buffer may be overwritten by the multicast of the next step.
        named_bar_sync(1, 256);
        if (warp == 0 && lane < TC_NC) mbar_arrive_cluster(mapa_u32(smem_u32(&bars->h_written), (uint32_t)lane));
        if (SAVE) {
          // Saved gates / cell states are not needed by the h exchange: they go out after the publish, so that the
          // release above does not wait for them.  The gates are evaluated again from the accumulators (still intact
          // until the next step's MMAs) -- cheaper than holding 80 packed values per thread across the publish.
#pragma unroll
          for (int c = 0; c < 4; ++c) {
            const float* bs = bias_s + c * 64;
#pragma unroll
            for (int h = 0; h < 2; ++h) {
              const int m = r0 + 8 * h;
              if ((long)tile_c * 128 + m >= p.B) continue;
              // saved state, SoA at 32-byte granularity: [(t, tile, 32-unit block fr, row quadrant)][piece = gate*2 +
              // h16][row & 31][16], unit = 32 fr + 16 h16 + e; this chunk is fr = 2 rank + c / 2, h16 = c % 2
              const long blk = (((long)t * p.n_tiles_cap + tile_c) * 8 + 2 * (int)rank + (c >> 1)) * 4 + (m >> 5);
#pragma unroll
              for (int q = 0; q < 2; ++q) {
                const int jj = 8 * q + 2 * cq;
                float gv[4][2];
                fwd_gates(acc[c >> 1] + 32 * (c & 1), bs, h, q, jj, gv);
                __nv_bfloat16* gp = p.gates + (blk * 8 + (c & 1)) * 512 + (m & 31) * 16 + jj;
#pragma unroll
                for (int g = 0; g < 4; ++g)
                  *reinterpret_cast<uint32_t*>(gp + g * 1024) = pack_bf16x2(gv[g][0], gv[g][1]);
                *reinterpret_cast<uint32_t*>(p.cst + (blk * 2 + (c & 1)) * 512 + (m & 31) * 16 + jj) =
                    pack_bf16x2(cstate[c][h][q][0], cstate[c][h][q][1]);
              }
            }
          }
        }
      }
    }
  }
  __syncwarp();
  cluster_sync_all();          // nobody leaves while peers may still multicast into / arrive on this CTA
}

// =============================================================================================
// Fused head: BN(inference affine) -> Dropout -> Dense -> weighted-MSE loss -> (training) all head gradients
// and dLoss/dh.  One warp per [b,t] row, H = 256 (8 hidden units per lane), n_outputs <= 16.
// (models/point_estimate/rnn_point_estimate.py:88-89,105; model_utils/losses.py:55-135; SURVEY App. A.2-A.4)
// =============================================================================================
struct HeadParams {
  int B, T, O, target_idx, train;
  const __nv_bfloat16* xh;
  const float *gamma, *beta, *mean, *var;
  float eps;
  const float *Wo, *bo;
  const float* y;
  const float* denom;
  float p1, p2;
  int use_dropout;
  DropoutKey key;
  int64_t row0;
  float* preds;
  __nv_bfloat16* dhout;
  float* dpred;         // [B*T][16] dLoss/dpred (training), consumed by head_wgrad_kernel
  float* partial;       // [gridDim.x][HEAD_PART]
};

constexpr int HEAD_PART = 2 * TC_H + TC_OPAD + 16;   // dgamma | dbeta | dbo | s0 s1 s2 (per CTA of the fused pass)
constexpr int HWG_PART = TC_H * TC_OPAD;              // dWo partial per CTA of the weight-gradient pass
constexpr int HWG_ROWS = 32;                          // rows staged per tile

// Thread-per-row head over TMA-staged tiles: a CTA takes 128 windows of one time step (the 128 x 256 bf16 h tile
// arrives as four SWIZZLE_128B boxes), every thread owns one row: y = Dropout(BN(h)) on the fly, pred = y*Wo + bo
// with Wo broadcast from shared memory (no cross-lane traffic), loss terms, dLoss/dpred, dy = dpred*Wo^T, dLoss/dh
// written in the backward kernel's SoA layout; dgamma/dbeta need a cross-row sum per column, done with a 31-shuffle
// reduce-scatter per group of 32 columns.
constexpr int HROWS_SMEM = 65536 + 1024 + 256;

template <bool TRAIN>
__global__ void __launch_bounds__(128, 2) head_rows_kernel(HeadParams p, const __grid_constant__ CUtensorMap tm_h,
                                                          int n_btiles, int n_tiles_cap) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* tile = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint64_t* bar = reinterpret_cast<uint64_t*>(tile + 65536);
  __shared__ __align__(16) float Wo_s[TC_H * TC_OPAD];
  __shared__ __align__(16) float bn_s[4][TC_H];      // gamma*inv | beta - gamma*mean*inv | mean | inv
  __shared__ float red_s[HEAD_PART];
  const int tid = threadIdx.x, lane = tid & 31, wq = tid >> 5;
  for (int j = tid; j < TC_H; j += 128) {
    const float iv = 1.0f / sqrtf(p.var[j] + p.eps);
    bn_s[0][j] = p.gamma[j] * iv;
    bn_s[1][j] = p.beta[j] - p.gamma[j] * p.mean[j] * iv;
    bn_s[2][j] = p.mean[j];
    bn_s[3][j] = iv;
  }
  for (int i = tid; i < TC_H * TC_OPAD; i += 128) {
    const int j = i / TC_OPAD, k = i % TC_OPAD;
    Wo_s[i] = (k < p.O) ? p.Wo[j * p.O + k] : 0.f;
  }
  for (int i = tid; i < HEAD_PART; i += 128) red_s[i] = 0.f;
  if (tid == 0) {
    mbar_init(bar, 1);
    fence_mbar_init();
  }
  __syncthreads();
  float c_all = 0.f, c_last = 0.f, c_tar = 0.f;
  if (TRAIN) {
    const float Bg = p.denom[0], Mg = p.denom[1];
    c_all = (1.f - p.p1) * (1.f - p.p2) / ((float)p.O * Mg);
    c_last = (1.f - p.p1) * p.p2 / (Bg * (float)p.O);
    c_tar = p.p1 / Bg;
  }
  float s0 = 0.f, s1 = 0.f, s2 = 0.f;
  float accbo[TC_OPAD];
#pragma unroll
  for (int k = 0; k < TC_OPAD; ++k) accbo[k] = 0.f;
  const int sw = tid & 7;
  const int nq = TC_H / 4;
  uint32_t phase = 0;
  const int n_tiles = p.T * n_btiles;
  for (int ti = blockIdx.x; ti < n_tiles; ti += gridDim.x) {
    const int t = ti / n_btiles, bt = ti % n_btiles;
    const long b = (long)bt * 128 + tid;
    const bool valid = b < p.B;
    if (tid == 0) {
      mbar_arrive_expect_tx(bar, 65536);
      for (int kb = 0; kb < 4; ++kb)
        tma_load_2d(tile + kb * 16384, &tm_h, bar, (t + 1) * TC_XH_LD + kb * 64, bt * 128);
    }
    const long r = b * p.T + t;
    float yt[TC_OPAD];
#pragma unroll
    for (int k = 0; k < TC_OPAD; ++k) yt[k] = 0.f;
    if (p.y && valid) {
      for (int k = 0; k < p.O; ++k) yt[k] = p.y[r * p.O + k];
    }
    mbar_wait(bar, phase);
    phase ^= 1;
    const uint8_t* hrow = tile + tid * 128;
    float pr[TC_OPAD];
#pragma unroll
    for (int k = 0; k < TC_OPAD; ++k) pr[k] = (k < p.O) ? p.bo[k] : 0.f;
#pragma unroll 4
    for (int c = 0; c < 32; ++c) {
      const uint4 raw = *reinterpret_cast<const uint4*>(hrow + (c >> 3) * 16384 + (((c & 7) ^ sw) << 4));
      const uint32_t hw[4] = {raw.x, raw.y, raw.z, raw.w};
      float dm[8];
      if (p.use_dropout) {
        const uint64_t qbase = ((uint64_t)(p.row0 + b) * p.T + t) * nq + c * 2;
        dropout_quad(p.key, qbase, dm);
        dropout_quad(p.key, qbase + 1, dm + 4);
      } else {
#pragma unroll
        for (int e = 0; e < 8; ++e) dm[e] = 1.f;
      }
#pragma unroll
      for (int e = 0; e < 8; ++e) {
        const int j = c * 8 + e;
        const float hv = (e & 1) ? bf16_hi(hw[e >> 1]) : bf16_lo(hw[e >> 1]);
        const float yv = fmaf(bn_s[0][j], hv, bn_s[1][j]) * dm[e];
        const float4* w4 = reinterpret_cast<const float4*>(Wo_s + j * TC_OPAD);
#pragma unroll
        for (int kk = 0; kk < 4; ++kk) {
          const float4 w = w4[kk];
          pr[4 * kk + 0] = fmaf(yv, w.x, pr[4 * kk + 0]);
          pr[4 * kk + 1] = fmaf(yv, w.y, pr[4 * kk + 1]);
          pr[4 * kk + 2] = fmaf(yv, w.z, pr[4 * kk + 2]);
          pr[4 * kk + 3] = fmaf(yv, w.w, pr[4 * kk + 3]);
        }
      }
    }
    if (p.preds && valid) {
      for (int k = 0; k < p.O; ++k) p.preds[r * p.O + k] = pr[k];
    }
    if (p.y) {
      bool any = false;
#pragma unroll
      for (int k = 0; k < TC_OPAD; ++k) any |= (yt[k] != 0.0f);          // losses.py:72
      const float mk = (any && valid) ? 1.f : 0.f;
      const bool last = (t == p.T - 1);
      float dp[TC_OPAD];
#pragma unroll
      for (int k = 0; k < TC_OPAD; ++k) {
        const float d = (k < p.O && valid) ? (pr[k] * mk - yt[k]) : 0.f;  // losses.py:75
        const float d2 = d * d;
        s2 += d2;
        float coef = c_all;
        if (last) {
          s1 += d2;
          coef += c_last;
          if (k == p.target_idx) {
            s0 += d2;
            coef += c_tar;
          }
        }
        dp[k] = TRAIN ? 2.f * d * coef * mk : 0.f;
        if (TRAIN) accbo[k] += dp[k];
      }
      if (TRAIN) {
        if (valid) {
#pragma unroll
          for (int k4 = 0; k4 < TC_OPAD; k4 += 4)
            *reinterpret_cast<float4*>(p.dpred + r * TC_OPAD + k4) = make_float4(dp[k4], dp[k4 + 1], dp[k4 + 2], dp[k4 + 3]);
        }
        // dLoss/dh in the backward kernel's layout: [t][tile][rank r'][warp][chunk][lane][16]
        __nv_bfloat16* dh_base = p.dhout + ((((long)t * n_tiles_cap + bt) * 4) * 4 + wq) * 4 * 32 * 16 + lane * 16;
#pragma unroll 1
        for (int grp = 0; grp < 8; ++grp) {          // 32 columns per group
          float dd[32], gd[32];
#pragma unroll
          for (int cc = 0; cc < 4; ++cc) {
            const int c = grp * 4 + cc;
            const uint4 raw = *reinterpret_cast<const uint4*>(hrow + (c >> 3) * 16384 + (((c & 7) ^ sw) << 4));
            const uint32_t hw[4] = {raw.x, raw.y, raw.z, raw.w};
            float dm[8];
            if (p.use_dropout) {
              const uint64_t qbase = ((uint64_t)(p.row0 + b) * p.T + t) * nq + c * 2;
              dropout_quad(p.key, qbase, dm);
              dropout_quad(p.key, qbase + 1, dm + 4);
            } else {
#pragma unroll
              for (int e = 0; e < 8; ++e) dm[e] = 1.f;
            }
#pragma unroll
            for (int e = 0; e < 8; ++e) {
              const int j = c * 8 + e;
              const float hv = (e & 1) ? bf16_hi(hw[e >> 1]) : bf16_lo(hw[e >> 1]);
              const float4* w4 = reinterpret_cast<const float4*>(Wo_s + j * TC_OPAD);
              float sacc = 0.f;
#pragma unroll
              for (int kk = 0; kk < 4; ++kk) {
                const float4 w = w4[kk];
                sacc = fmaf(dp[4 * kk + 0], w.x, sacc);
                sacc = fmaf(dp[4 * kk + 1], w.y, sacc);
                sacc = fmaf(dp[4 * kk + 2], w.z, sacc);
                sacc = fmaf(dp[4 * kk + 3], w.w, sacc);
              }
              const float d_ = sacc * dm[e];                       // through Dropout
              dd[cc * 8 + e] = d_;
              gd[cc * 8 + e] = d_ * (hv - bn_s[2][j]) * bn_s[3][j];
            }
          }
          // dLoss/dh = dd * gamma * inv -> two 16-unit chunks of this group
          if (valid) {
#pragma unroll
            for (int hh = 0; hh < 2; ++hh) {
              uint32_t pk[8];
#pragma unroll
              for (int e = 0; e < 8; ++e) {
                const int jj = hh * 16 + 2 * e;
                pk[e] = pack_bf16x2(dd[jj] * bn_s[0][grp * 32 + jj], dd[jj + 1] * bn_s[0][grp * 32 + jj + 1]);
              }
              const int c16 = grp * 2 + hh;                         // 16-unit chunk 0..15: rank r' = c16/4, chunk c16%4
              st_global_v8(dh_base + ((long)(c16 >> 2) * 4 * 4 + (c16 & 3)) * 32 * 16, pk);
            }
          }
          // column sums over the warp's 32 rows: reduce-scatter butterfly, lane l ends with column perm(l)
#pragma unroll
          for (int off = 16; off >= 1; off >>= 1) {
#pragma unroll
            for (int i = 0; i < off; ++i) {
              const bool up = (lane & off) != 0;
              const float sd = up ? dd[i] : dd[i + off];
              const float kd = up ? dd[i + off] : dd[i];
              dd[i] = kd + __shfl_xor_sync(0xffffffffu, sd, off);
              const float sg = up ? gd[i] : gd[i + off];
              const float kg = up ? gd[i + off] : gd[i];
              gd[i] = kg + __shfl_xor_sync(0xffffffffu, sg, off);
            }
          }
          // lane's column within the group: bit b of lane selects +2^b  (lane bit4 -> +16 ... bit0 -> +1)
          atomicAdd(&red_s[TC_H + grp * 32 + lane], dd[0]);
          atomicAdd(&red_s[grp * 32 + lane], gd[0]);
        }
      }
    }
    __syncthreads();        // everyone is done with the tile before it is overwritten
  }
  if (p.y) {
    // block-level sums of the loss terms and dbo
    s0 = warp_sum(s0); s1 = warp_sum(s1); s2 = warp_sum(s2);
#pragma unroll
    for (int k = 0; k < TC_OPAD; ++k) accbo[k] = warp_sum(accbo[k]);
    if (lane == 0) {
      atomicAdd(&red_s[2 * TC_H + TC_OPAD + 0], s0);
      atomicAdd(&red_s[2 * TC_H + TC_OPAD + 1], s1);
      atomicAdd(&red_s[2 * TC_H + TC_OPAD + 2], s2);
      if (TRAIN)
        for (int k = 0; k < TC_OPAD; ++k) atomicAdd(&red_s[2 * TC_H + k], accbo[k]);
    }
    __syncthreads();
    for (int i = tid; i < HEAD_PART; i += 128) p.partial[(long)i * gridDim.x + blockIdx.x] = red_s[i];
  }
}

// Tensor-core head (dropout off): with y = a*h + b (BN inference affine) the Dense layer folds to
//   pred = h * (diag(a) Wo) + (bo + b Wo)
// a wgmma on the TMA-staged h tile (K-major SW128, exactly the layout the recurrence uses): 2 x 16 x (M64 N16 K16).
// Threads own one row each for the loss terms and dpred, staged as a 128 x 32 bf16 tile (SW64).  Training: that tile
// feeds h^T dpred (MN-major MMAs, accumulated in registers across tiles -> dWo, dgamma) and goes to HBM by TMA store for the
// backward recurrence, which forms dLoss/dh = dpred (Wo a)^T on its own tensor cores; colsum(dpred) -> dbo, dbeta.
struct HeadTcWeights {
  const __nv_bfloat16* WoTp;   // [16][256]  a_j * Wo[j][n]
  const float* bop;            // [16]       bo + sum_j b_j Wo[j][k]
};

__device__ __forceinline__ void pack_head_body(int bid, int O, const float* __restrict__ Wo, const float* __restrict__ bo,
                                 const float* __restrict__ gamma, const float* __restrict__ beta,
                                 const float* __restrict__ mean, const float* __restrict__ var, float eps,
                                 __nv_bfloat16* __restrict__ WoTp, __nv_bfloat16* __restrict__ WoSp,
                                 float* __restrict__ bop) {
  const int idx = bid * blockDim.x + threadIdx.x;
  if (idx < TC_OPAD * TC_H) {
    const int n = idx / TC_H, j = idx % TC_H;
    const float a = gamma[j] / sqrtf(var[j] + eps);
    WoTp[idx] = __float2bfloat16(n < O ? a * Wo[j * O + n] : 0.f);
  }
  if (idx < TC_H * 32) {
    const int j = idx / 32, k = idx % 32;
    WoSp[idx] = __float2bfloat16(k < O ? Wo[j * O + k] * gamma[j] / sqrtf(var[j] + eps) : 0.f);
  }
  // folded bias: block k (< 16) reduces over its 256 threads = 256 hidden units
  if (bid < TC_OPAD) {
    __shared__ float red[8];
    const int k = bid, j = threadIdx.x;
    float v = 0.f;
    if (k < O) {
      const float iv = 1.0f / sqrtf(var[j] + eps);
      v = (beta[j] - gamma[j] * mean[j] * iv) * Wo[j * O + k];
    }
    v = warp_sum(v);
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
    __syncthreads();
    if (threadIdx.x == 0) {
      float t = (k < O) ? bo[k] : 0.f;
      for (int w = 0; w < 8; ++w) t += red[w];
      bop[k] = t;
    }
  }
}

// Ubk[r][n][k'] = U[n][g*H + 64r + 16jb + jj], k' = 64jb + 16g + jj   (K-slices of U for the backward recurrence)
__device__ __forceinline__ void pack_ubk_body(int bid, const float* __restrict__ U, __nv_bfloat16* __restrict__ Ubk) {
  const long idx = (long)bid * blockDim.x + threadIdx.x;
  if (idx >= (long)4 * TC_H * TC_H) return;
  const int kp = (int)(idx % 256);
  const int n = (int)((idx / 256) % TC_H);
  const int r = (int)(idx / (256 * TC_H));
  const int jb = kp / 64, g = (kp % 64) / 16, jj = kp % 16;
  Ubk[idx] = __float2bfloat16(U[(long)n * 4 * TC_H + g * TC_H + 64 * r + 16 * jb + jj]);
}

// All weight repacking of one optimizer step in ONE launch: block ranges [0,nb_w) forward slices, [nb_w,nb_w+nb_h)
// head, the rest the backward K-slices (nb_u = 0 on a forward-only handle).
struct PackArgs {
  int I, O, nb_w, nb_h, nb_u;
  float eps;
  const float *W, *U, *bias, *Wo, *bo, *gamma, *beta, *mean, *var;
  __nv_bfloat16 *Up, *Wp, *Ubk, *WoTp, *WoSp;
  float *biasp, *bop;
};

__global__ void __launch_bounds__(256) pack_all_kernel(PackArgs a) {
  pdl_sync();
  const int bid = blockIdx.x;
  if (bid < a.nb_w) {
    pack_weights_body(bid, a.I, a.W, a.U, a.bias, a.Up, a.Wp, a.biasp);
  } else if (bid < a.nb_w + a.nb_h) {
    pack_head_body(bid - a.nb_w, a.O, a.Wo, a.bo, a.gamma, a.beta, a.mean, a.var, a.eps, a.WoTp, a.WoSp, a.bop);
  } else {
    pack_ubk_body(bid - a.nb_w - a.nb_h, a.U, a.Ubk);
  }
}

constexpr uint32_t HT_TILE = 0;            // 4 k-blocks x [128 x 128 B]
constexpr uint32_t HT_WOT = 65536;         // 4 k-blocks x [16 x 128 B]
constexpr uint32_t HT_PRED = 73728;        // [128][17] fp32: pred rows, fragment -> one row per thread
constexpr uint32_t HT_DP = 90112;          // [128 x 64 B]
constexpr uint32_t HT_BARS = 98304;
constexpr int HT_SMEM = HT_BARS + 128 + 1024;
constexpr int HT_THREADS = 160;            // warps 0-3: MMA warpgroup, one row per thread; warp 4: TMA
constexpr int HT_PRED_LD = 17;

struct HtBars {
  uint64_t wt_full, tile_full, tile_free;
};

template <bool TRAIN>
__global__ void __launch_bounds__(HT_THREADS, 2)
    head_tc_kernel(HeadParams p, HeadTcWeights w, const __grid_constant__ CUtensorMap tm_h,
                   const __grid_constant__ CUtensorMap tm_wot, const __grid_constant__ CUtensorMap tm_dpb, int n_btiles, int n_tiles_cap,
                   float* __restrict__ wpartial) {
  pdl_sync();
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  HtBars* bars = reinterpret_cast<HtBars*>(smem + HT_BARS);
  float* pred_s = reinterpret_cast<float*>(smem + HT_PRED);
  __shared__ __align__(16) float bn_s[3][TC_H];      // gamma*inv | mean | inv
  __shared__ float red_s[HEAD_PART];
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  for (int j = tid; j < TC_H; j += HT_THREADS) {
    const float iv = 1.0f / sqrtf(p.var[j] + p.eps);
    bn_s[0][j] = p.gamma[j] * iv;
    bn_s[1][j] = p.mean[j];
    bn_s[2][j] = iv;
  }
  for (int i = tid; i < HEAD_PART; i += HT_THREADS) red_s[i] = 0.f;
  // zero the dpred staging tile once (padding columns stay zero)
  for (int i = tid; i < 128 * 64 / 16; i += HT_THREADS) reinterpret_cast<uint4*>(smem + HT_DP)[i] = make_uint4(0, 0, 0, 0);
  if (tid == 0) {
    mbar_init(&bars->wt_full, 1);
    mbar_init(&bars->tile_full, 1);
    mbar_init(&bars->tile_free, 1);
    fence_mbar_init();
  }
  fence_proxy_async_smem();
  __syncthreads();
  const int n_tiles = p.T * n_btiles;

  if (warp == 4) {
    if (lane == 0) {
      mbar_arrive_expect_tx(&bars->wt_full, 8192);
      for (int kb = 0; kb < 4; ++kb) tma_load_2d(smem + HT_WOT + kb * 2048, &tm_wot, &bars->wt_full, kb * 64, 0);
      uint32_t n = 0;
      for (int ti = blockIdx.x; ti < n_tiles; ti += gridDim.x, ++n) {
        const int t = ti / n_btiles, bt = ti % n_btiles;
        if (n > 0) mbar_wait(&bars->tile_free, (n - 1) & 1);
        mbar_arrive_expect_tx(&bars->tile_full, 65536);
        for (int kb = 0; kb < 4; ++kb)
          tma_load_2d(smem + HT_TILE + kb * 16384, &tm_h, &bars->tile_full, (t + 1) * TC_XH_LD + kb * 64, bt * 128);
      }
    }
  } else {
    const int mrow = tid;                   // row of the tile this thread owns
    const int fw = warp, cq = lane & 3;     // accumulator fragment: rows 16 fw + lane / 4 (+ 8) of each 64-row half
    float c_all = 0.f, c_last = 0.f, c_tar = 0.f;
    if (TRAIN) {
      const float Bg = p.denom[0], Mg = p.denom[1];
      c_all = (1.f - p.p1) * (1.f - p.p2) / ((float)p.O * Mg);
      c_last = (1.f - p.p1) * p.p2 / (Bg * (float)p.O);
      c_tar = p.p1 / Bg;
    }
    float bop[TC_OPAD];
#pragma unroll
    for (int k = 0; k < TC_OPAD; ++k) bop[k] = w.bop[k];
    float s0 = 0.f, s1 = 0.f, s2 = 0.f;
    float accbo[TC_OPAD];
#pragma unroll
    for (int k = 0; k < TC_OPAD; ++k) accbo[k] = 0.f;
    // this CTA's sum over its tiles of h^T dpred: hidden units 64 mq .. 64 mq + 63 (M) x 16 outputs (N)
    float accw[4][8];
#pragma unroll
    for (int mq = 0; mq < 4; ++mq)
#pragma unroll
      for (int i = 0; i < 8; ++i) accw[mq][i] = 0.f;
    mbar_wait(&bars->wt_full, 0);
    uint32_t n = 0;
    for (int ti = blockIdx.x; ti < n_tiles; ti += gridDim.x, ++n) {
      const int t = ti / n_btiles, bt = ti % n_btiles;
      const long b = (long)bt * 128 + mrow;
      const bool valid = b < p.B;
      const long r = b * p.T + t;
      float yt[TC_OPAD];
#pragma unroll
      for (int k = 0; k < TC_OPAD; ++k) yt[k] = 0.f;
      if (p.y && valid) {
#pragma unroll
        for (int k = 0; k < TC_OPAD; ++k)
          if (k < p.O) yt[k] = p.y[r * p.O + k];
      }
      mbar_wait(&bars->tile_full, n & 1);
      // pred = h (diag(a) Wo): two m64 x n16 halves, K = 256
      float ap[2][8];
      wgmma_fence();
#pragma unroll
      for (int mh = 0; mh < 2; ++mh)
#pragma unroll
        for (int kb = 0; kb < 4; ++kb)
#pragma unroll
          for (int k16 = 0; k16 < 4; ++k16) {
            const uint64_t da = make_smem_desc(smem_u32(smem + HT_TILE + kb * 16384 + mh * 8192) + k16 * 32, 0, 1024,
                                               LAYOUT_SW128);
            const uint64_t db = make_smem_desc(smem_u32(smem + HT_WOT + kb * 2048) + k16 * 32, 0, 1024, LAYOUT_SW128);
            wgmma_m64n16k16<0, 0>(ap[mh], da, db, (kb | k16) != 0);
          }
      wgmma_commit();
      wgmma_wait<0>();
      fence_regs(ap[0]);
      fence_regs(ap[1]);
#pragma unroll
      for (int mh = 0; mh < 2; ++mh)
#pragma unroll
        for (int i = 0; i < 8; ++i)
          pred_s[(64 * mh + 16 * fw + (lane >> 2) + 8 * ((i >> 1) & 1)) * HT_PRED_LD + 8 * (i >> 2) + 2 * cq + (i & 1)] =
              ap[mh][i];
      named_bar_sync(1, 128);
      float pr[TC_OPAD];
#pragma unroll
      for (int k = 0; k < TC_OPAD; ++k) pr[k] = pred_s[mrow * HT_PRED_LD + k] + bop[k];
      if (p.preds && valid) {
#pragma unroll
        for (int k = 0; k < TC_OPAD; ++k)
          if (k < p.O) p.preds[r * p.O + k] = pr[k];
      }
      if (p.y) {
        bool any = false;
#pragma unroll
        for (int k = 0; k < TC_OPAD; ++k) any |= (yt[k] != 0.0f);          // losses.py:72
        const float mk = (any && valid) ? 1.f : 0.f;
        const bool last = (t == p.T - 1);
        float dp[TC_OPAD];
#pragma unroll
        for (int k = 0; k < TC_OPAD; ++k) {
          const float d = (k < p.O && valid) ? (pr[k] * mk - yt[k]) : 0.f;  // losses.py:75
          const float d2 = d * d;
          s2 += d2;
          float coef = c_all;
          if (last) {
            s1 += d2;
            coef += c_last;
            if (k == p.target_idx) {
              s0 += d2;
              coef += c_tar;
            }
          }
          dp[k] = TRAIN ? 2.f * d * coef * mk : 0.f;
          if (TRAIN) accbo[k] += dp[k];
        }
        if (TRAIN) {
          if (valid && p.dpred) {        // fp32 copy: only the dropout path's SIMT weight-gradient kernel reads it
#pragma unroll
            for (int k4 = 0; k4 < TC_OPAD; k4 += 4)
              *reinterpret_cast<float4*>(p.dpred + r * TC_OPAD + k4) = make_float4(dp[k4], dp[k4 + 1], dp[k4 + 2], dp[k4 + 3]);
          }
          // the TMA store of the previous tile's dpred has read the staging tile (the MMAs that read it are complete)
          if (n > 0 && tid == 0) bulk_wait_group_read0();
          named_bar_sync(1, 128);
          // dpred row -> [128 x 64 B] tile, SWIZZLE_64B: chunk c of row m at m*64 + ((c ^ ((m>>1)&3)) << 4)
          uint8_t* drow = smem + HT_DP + mrow * 64;
          const int s64 = (mrow >> 1) & 3;
          *reinterpret_cast<uint4*>(drow + ((0 ^ s64) << 4)) =
              make_uint4(pack_bf16x2(dp[0], dp[1]), pack_bf16x2(dp[2], dp[3]), pack_bf16x2(dp[4], dp[5]), pack_bf16x2(dp[6], dp[7]));
          *reinterpret_cast<uint4*>(drow + ((1 ^ s64) << 4)) =
              make_uint4(pack_bf16x2(dp[8], dp[9]), pack_bf16x2(dp[10], dp[11]), pack_bf16x2(dp[12], dp[13]), pack_bf16x2(dp[14], dp[15]));
          fence_proxy_async_smem();
          named_bar_sync(1, 128);
          // the staged dLoss/dpred tile also goes to HBM as it is (128 x 64 B, SW64): the backward recurrence adds
          // dpred (Wo gamma inv)^T for its own hidden units on its tensor cores
          if (tid == 0) {
            tma_store_2d(&tm_dpb, smem + HT_DP, 0, (t * n_tiles_cap + bt) * 128);
            bulk_commit_group();
          }
          // dWo' += h^T dpred: A = the h tile read MN-major (hidden unit = M), B = the dpred tile read MN-major,
          // K = the 128 rows
          wgmma_fence();
#pragma unroll
          for (int mq = 0; mq < 4; ++mq)
#pragma unroll
            for (int k16 = 0; k16 < 8; ++k16) {
              const uint64_t wa = make_smem_desc(smem_u32(smem + HT_TILE + mq * 16384) + k16 * 2048, 16384, 1024,
                                                 LAYOUT_SW128);
              const uint64_t wb = make_smem_desc(smem_u32(smem + HT_DP) + k16 * 1024, 0, 512, LAYOUT_SW64);
              wgmma_m64n16k16<1, 1>(accw[mq], wa, wb, 1);
            }
          wgmma_commit();
          wgmma_wait<0>();
#pragma unroll
          for (int mq = 0; mq < 4; ++mq) fence_regs(accw[mq]);
          // nothing else per tile: dLoss/dh is formed by the backward recurrence from the dpred tile (lstm_bwd_tc_kernel
          // <FUSED>), dgamma / dbeta by head_fold_kernel from h^T dpred and colsum(dpred)
        }
      }
      named_bar_sync(1, 128);               // the tile and the pred rows have been read by everybody
      if (tid == 0) mbar_arrive(&bars->tile_free);
    }
    if (p.y) {
      s0 = warp_sum(s0); s1 = warp_sum(s1); s2 = warp_sum(s2);
#pragma unroll
      for (int k = 0; k < TC_OPAD; ++k) accbo[k] = warp_sum(accbo[k]);
      if (lane == 0) {
        atomicAdd(&red_s[2 * TC_H + TC_OPAD + 0], s0);
        atomicAdd(&red_s[2 * TC_H + TC_OPAD + 1], s1);
        atomicAdd(&red_s[2 * TC_H + TC_OPAD + 2], s2);
        if (TRAIN)
          for (int k = 0; k < TC_OPAD; ++k) atomicAdd(&red_s[2 * TC_H + k], accbo[k]);
      }
    }
    if (TRAIN) {
      // this CTA's h^T dpred, [hidden unit][16]
      float* wp = wpartial + (long)blockIdx.x * HWG_PART;
#pragma unroll
      for (int mq = 0; mq < 4; ++mq)
#pragma unroll
        for (int i = 0; i < 8; i += 2) {
          const int j = 64 * mq + 16 * fw + (lane >> 2) + 8 * ((i >> 1) & 1);
          *reinterpret_cast<float2*>(wp + j * TC_OPAD + 8 * (i >> 2) + 2 * cq) = make_float2(accw[mq][i], accw[mq][i + 1]);
        }
      if (tid == 0) bulk_wait_group0();
    }
  }
  __syncthreads();
  if (p.y)
    for (int i = tid; i < HEAD_PART; i += HT_THREADS) p.partial[(long)i * gridDim.x + blockIdx.x] = red_s[i];
}

// dWo[j][k] = sum_r y[r][j] * dpred[r][k] with y = Dropout(BN(h)) recomputed from h: CTA tiles of 32 rows staged in
// shared memory, thread (j-group of 4, k-group of 4) keeps a 4x4 block of the 256 x 16 result.
__global__ void __launch_bounds__(256, 2) head_wgrad_kernel(HeadParams p, float* __restrict__ wpartial) {
  __shared__ __align__(16) float y_s[HWG_ROWS][TC_H];
  __shared__ __align__(16) float dp_s[HWG_ROWS][TC_OPAD];
  __shared__ __align__(16) float bn_s[2][TC_H];
  const int tid = threadIdx.x;
  for (int j = tid; j < TC_H; j += 256) {
    const float iv = 1.0f / sqrtf(p.var[j] + p.eps);
    bn_s[0][j] = p.gamma[j] * iv;
    bn_s[1][j] = p.beta[j] - p.gamma[j] * p.mean[j] * iv;
  }
  const int jg = tid >> 2, kg = tid & 3;
  float acc[4][4];
#pragma unroll
  for (int a = 0; a < 4; ++a)
#pragma unroll
    for (int b = 0; b < 4; ++b) acc[a][b] = 0.f;
  const long rows = (long)p.B * p.T;
  const int nq = TC_H / 4;
  __syncthreads();
  for (long r0 = (long)blockIdx.x * HWG_ROWS; r0 < rows; r0 += (long)gridDim.x * HWG_ROWS) {
    // stage: 32 rows x 256 cols, each thread converts 4 x (8 bf16)
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const int idx = tid + 256 * i;            // 0..1023 = 32 rows x 32 chunks of 8
      const int rr = idx >> 5, ch = idx & 31;
      const long r = r0 + rr;
      float v[8];
      if (r < rows) {
        const long b = r / p.T;
        const int t = (int)(r % p.T);
        const uint4 raw = *reinterpret_cast<const uint4*>(p.xh + (b * (p.T + 1) + t + 1) * TC_XH_LD + ch * 8);
        const uint32_t hw[4] = {raw.x, raw.y, raw.z, raw.w};
        float dm[8];
        if (p.use_dropout) {
          const uint64_t qbase = ((uint64_t)(p.row0 + b) * p.T + t) * nq + ch * 2;
          dropout_quad(p.key, qbase, dm);
          dropout_quad(p.key, qbase + 1, dm + 4);
        } else {
#pragma unroll
          for (int e = 0; e < 8; ++e) dm[e] = 1.f;
        }
#pragma unroll
        for (int e = 0; e < 4; ++e) {
          v[2 * e] = fmaf(bn_s[0][ch * 8 + 2 * e], bf16_lo(hw[e]), bn_s[1][ch * 8 + 2 * e]) * dm[2 * e];
          v[2 * e + 1] = fmaf(bn_s[0][ch * 8 + 2 * e + 1], bf16_hi(hw[e]), bn_s[1][ch * 8 + 2 * e + 1]) * dm[2 * e + 1];
        }
      } else {
#pragma unroll
        for (int e = 0; e < 8; ++e) v[e] = 0.f;
      }
      *reinterpret_cast<float4*>(&y_s[rr][ch * 8]) = make_float4(v[0], v[1], v[2], v[3]);
      *reinterpret_cast<float4*>(&y_s[rr][ch * 8 + 4]) = make_float4(v[4], v[5], v[6], v[7]);
    }
    for (int idx = tid; idx < HWG_ROWS * TC_OPAD; idx += 256) {
      const long r = r0 + idx / TC_OPAD;
      dp_s[idx / TC_OPAD][idx % TC_OPAD] = (r < rows) ? p.dpred[r * TC_OPAD + idx % TC_OPAD] : 0.f;
    }
    __syncthreads();
#pragma unroll 8
    for (int rr = 0; rr < HWG_ROWS; ++rr) {
      const float4 yv = *reinterpret_cast<const float4*>(&y_s[rr][jg * 4]);
      const float4 dv = *reinterpret_cast<const float4*>(&dp_s[rr][kg * 4]);
      const float ya[4] = {yv.x, yv.y, yv.z, yv.w};
      const float da[4] = {dv.x, dv.y, dv.z, dv.w};
#pragma unroll
      for (int a = 0; a < 4; ++a)
#pragma unroll
        for (int b = 0; b < 4; ++b) acc[a][b] = fmaf(ya[a], da[b], acc[a][b]);
    }
    __syncthreads();
  }
#pragma unroll
  for (int a = 0; a < 4; ++a)
#pragma unroll
    for (int b = 0; b < 4; ++b)
      wpartial[(long)blockIdx.x * HWG_PART + (jg * 4 + a) * TC_OPAD + kg * 4 + b] = acc[a][b];
}

// Sums the per-CTA head partials (stored [value][cta]: one warp per value, lanes over CTAs, fixed order) and
// scatters them into the flat gradient vector / loss tail.  wpartial is [cta][256*16].
__global__ void head_reduce_kernel(int n_cta, const float* __restrict__ partial, int n_wcta,
                                   const float* __restrict__ wpartial, int O, int B, const float* denom, float p1,
                                   float p2, int train, float* __restrict__ gWo, float* __restrict__ gbo,
                                   float* __restrict__ ggamma, float* __restrict__ gbeta, float* __restrict__ out2) {
  pdl_sync();
  const int i = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;     // one warp per output value
  const int lane = threadIdx.x & 31;
  if (i < HWG_PART) {
    if (!train) return;
    const int j = i / TC_OPAD, k = i % TC_OPAD;
    double s = 0.0;
    for (int c = lane; c < n_wcta; c += 32) s += wpartial[(long)c * HWG_PART + i];
    s = warp_sum(s);
    if (lane == 0 && k < O) gWo[j * O + k] = (float)s;
    return;
  }
  const int q = i - HWG_PART;
  if (q >= HEAD_PART) return;
  double s = 0.0;
  for (int c = lane; c < n_cta; c += 32) s += partial[(long)q * n_cta + c];
  s = warp_sum(s);
  if (q < TC_H) {
    if (train && lane == 0) ggamma[q] = (float)s;
  } else if (q < 2 * TC_H) {
    if (train && lane == 0) gbeta[q - TC_H] = (float)s;
  } else if (q < 2 * TC_H + TC_OPAD) {
    const int k = q - 2 * TC_H;
    if (train && lane == 0 && k < O) gbo[k] = (float)s;
  } else if (q == 2 * TC_H + TC_OPAD) {
    // the three loss sums live in consecutive slots; this warp finishes the loss (losses.py:87-98)
    double s1 = 0.0, s2 = 0.0;
    for (int c = lane; c < n_cta; c += 32) {
      s1 += partial[(long)(q + 1) * n_cta + c];
      s2 += partial[(long)(q + 2) * n_cta + c];
    }
    s1 = warp_sum(s1);
    s2 = warp_sum(s2);
    if (lane == 0) {
      const double Bg = denom[0], Mg = denom[1];
      const double mse0 = s / Bg, mse1 = s1 / (Bg * O), mse2 = s2 / (Mg * O);
      out2[0] = (float)(p1 * mse0 + (1.0 - p1) * (p2 * mse1 + (1.0 - p2) * mse2));
      out2[1] = (float)mse0;
    }
  }
}

// tensor-core head, one thread per hidden unit j.  In: G = h^T dpred (in gWo), cs = colsum(dpred) (in gbo).
// With y = a_j h + c_j (a = gamma*inv, c = beta - gamma*mean*inv) and dy = dpred Wo^T:
//   dWo[j][k] = a_j G[j][k] + c_j cs[k]
//   dbeta_j   = sum_r dy[r][j]           = sum_k Wo[j][k] cs[k]
//   dgamma_j  = sum_r dy[r][j] xhat[r][j] = inv_j (sum_k Wo[j][k] G[j][k] - mean_j dbeta_j)
__global__ void head_fold_kernel(int O, float* __restrict__ gWo, const float* __restrict__ gbo,
                                 float* __restrict__ ggamma, float* __restrict__ gbeta, const float* __restrict__ Wo,
                                 const float* __restrict__ gamma, const float* __restrict__ beta,
                                 const float* __restrict__ mean, const float* __restrict__ var, float eps) {
  pdl_sync();
  const int j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= TC_H) return;
  const float iv = 1.0f / sqrtf(var[j] + eps);
  const float a = gamma[j] * iv, c = beta[j] - gamma[j] * mean[j] * iv;
  float db = 0.f, sg = 0.f;
  for (int k = 0; k < O; ++k) {
    const float w = Wo[j * O + k], g = gWo[j * O + k], cs = gbo[k];
    db = fmaf(w, cs, db);
    sg = fmaf(w, g, sg);
    gWo[j * O + k] = fmaf(a, g, c * cs);
  }
  gbeta[j] = db;
  ggamma[j] = iv * (sg - mean[j] * db);
}

// =============================================================================================
// Host side
// =============================================================================================
static bool tc_supported(const lfmq_config& c, char* why, size_t n) {
  if (c.rnn_cell != LFMQ_CELL_LSTM) { snprintf(why, n, "the bf16 tensor-core path is built for the LSTM cell only"); return false; }
  if (c.uq) { snprintf(why, n, "the bf16 tensor-core path is built for the point-estimate head only"); return false; }
  if (c.num_hidden != TC_H) { snprintf(why, n, "num_hidden must be 256 (got %d)", c.num_hidden); return false; }
  if (c.num_layers != 1) { snprintf(why, n, "num_layers must be 1 (got %d)", c.num_layers); return false; }
  if (c.n_inputs > 32) { snprintf(why, n, "n_inputs must be <= 32 (got %d)", c.n_inputs); return false; }
  if (c.n_outputs > TC_OPAD) { snprintf(why, n, "n_outputs must be <= 16 (got %d)", c.n_outputs); return false; }
  if (c.recurrent_dropout > 0.f) { snprintf(why, n, "recurrent_dropout is not built on the bf16 path"); return false; }
  return true;
}

bool tc_shape_supported(const lfmq_config& c) {
  char why[128];
  return tc_supported(c, why, sizeof(why));
}

void tc_layout(TcState& st, const lfmq_config& c, const TcParamOff& po, Carver& cv) {
  if (c.precision != LFMQ_PREC_BF16) return;
  char why[128];
  if (!tc_supported(c, why, sizeof(why))) return;   // tc_init reports the error
  if (!st.impl) st.impl = new TcImpl;
  TcImpl& m = *st.impl;
  const size_t B = (size_t)c.max_batch, T = (size_t)c.seq_len, H = TC_H;
  m.maxB = c.max_batch; m.T = c.seq_len; m.I = c.n_inputs; m.O = c.n_outputs;
  m.eps = c.bn_epsilon;
  m.train = !c.forward_only;
  m.xh = cv.take<__nv_bfloat16>(B * (T + 1) * TC_XH_LD);
  m.Up = cv.take<__nv_bfloat16>(4 * H * H);
  m.Wp = cv.take<__nv_bfloat16>(4 * H * 32);
  m.Ubk = cv.take<__nv_bfloat16>(4 * H * H);
  m.biasp = cv.take<float>(4 * H);
  m.WoTp = cv.take<__nv_bfloat16>(TC_OPAD * H);
  m.WoSp = cv.take<__nv_bfloat16>(H * 32);
  m.bop = cv.take<float>(TC_OPAD);
  m.n_sms = device_sm_count();
  m.head_ctas = m.n_sms * 2;
  m.head_wctas = m.n_sms * 2;
  m.head_part_elems = (size_t)m.head_ctas * HEAD_PART;
  m.head_part = cv.take<float>(m.head_part_elems);
  if (m.train) {
    const size_t Bt = (B + 127) / 128 * 128;      // saved state is blocked by 128-row tiles
    m.gates = cv.take<__nv_bfloat16>(Bt * T * 4 * H);
    m.cst = cv.take<__nv_bfloat16>(Bt * T * H);
    m.dz = cv.take<__nv_bfloat16>(B * (T + 1) * 4 * H);
    m.dhout = cv.take<__nv_bfloat16>(((B + 127) / 128 * 128) * T * H);
    m.dpred = cv.take<float>(B * T * TC_OPAD);
    m.dpb = cv.take<__nv_bfloat16>(T * ((B + 127) / 128) * 128 * 32);
    m.head_wpart = cv.take<float>((size_t)m.head_wctas * HWG_PART);
    m.wg_part_elems = (size_t)64 * 384 * 1024;
    m.wg_part = cv.take<float>(m.wg_part_elems);
  } else {
    m.gates = nullptr; m.cst = nullptr; m.dz = nullptr; m.dhout = nullptr; m.wg_part = nullptr;
    m.dpred = nullptr; m.head_wpart = nullptr; m.dpb = nullptr;
    m.wg_part_elems = 0;
  }
  // offsets of the tensors in the flat parameter vector: the API layer's layout() is the one place that defines them
  m.oW = po.oW; m.oU = po.oU; m.ob = po.ob; m.ogamma = po.ogamma; m.obeta = po.obeta;
  m.oWo = po.oWo; m.obo = po.obo; m.omean = po.omean; m.ovar = po.ovar;
}

int tc_init(TcState& st, const lfmq_config& c) {
  if (c.precision != LFMQ_PREC_BF16) return 0;
  char why[128];
  if (!tc_supported(c, why, sizeof(why))) {
    LFMQ_SET_ERR("LFMQ_PREC_BF16 supports the H=256 single-layer forecaster only: %s; use LFMQ_PREC_FP32", why);
    return LFMQ_ERR_UNSUPPORTED;
  }
  TcImpl& m = *st.impl;
  const size_t B = (size_t)m.maxB, T = (size_t)m.T;
  LFMQ_CUDA_CHECK(cudaMemset(m.xh, 0, B * (T + 1) * TC_XH_LD * 2));
  if (m.dz) LFMQ_CUDA_CHECK(cudaMemset(m.dz, 0, B * (T + 1) * 4 * TC_H * 2));
  const uint64_t xh_row = (uint64_t)(T + 1) * TC_XH_LD;     // elements per batch row of the 2-D view
  int rc;
  if ((rc = encode_map_2d(&m.tm_h, m.xh, xh_row, B, xh_row * 2, 64, 32, CU_TENSOR_MAP_SWIZZLE_128B))) return rc;
  if ((rc = encode_map_2d(&m.tm_x, m.xh, xh_row, B, xh_row * 2, 32, 128, CU_TENSOR_MAP_SWIZZLE_64B))) return rc;
  if ((rc = encode_map_2d(&m.tm_h128, m.xh, xh_row, B, xh_row * 2, 64, 128, CU_TENSOR_MAP_SWIZZLE_128B))) return rc;
  if ((rc = encode_map_2d(&m.tm_wot, m.WoTp, TC_H, TC_OPAD, TC_H * 2, 64, 16, CU_TENSOR_MAP_SWIZZLE_128B))) return rc;
  if ((rc = encode_map_2d(&m.tm_wos, m.WoSp, 32, TC_H, 64, 32, 64, CU_TENSOR_MAP_SWIZZLE_64B))) return rc;
  if (m.dpb &&
      (rc = encode_map_2d(&m.tm_dpb, m.dpb, 32, (uint64_t)m.T * ((m.maxB + 127) / 128) * 128, 64, 32, 128,
                        CU_TENSOR_MAP_SWIZZLE_64B)))
    return rc;
  LFMQ_CUDA_CHECK(cudaFuncSetAttribute(head_tc_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, HT_SMEM));
  LFMQ_CUDA_CHECK(cudaFuncSetAttribute(head_tc_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, HT_SMEM));
  LFMQ_CUDA_CHECK(cudaFuncSetAttribute(head_rows_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, HROWS_SMEM));
  LFMQ_CUDA_CHECK(cudaFuncSetAttribute(head_rows_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, HROWS_SMEM));
  if ((rc = encode_map_2d(&m.tm_u, m.Up, TC_H, 4 * TC_H, TC_H * 2, 64, 256, CU_TENSOR_MAP_SWIZZLE_128B))) return rc;
  if ((rc = encode_map_2d(&m.tm_w, m.Wp, 32, 4 * TC_H, 64, 32, 256, CU_TENSOR_MAP_SWIZZLE_64B))) return rc;
  LFMQ_CUDA_CHECK(cudaFuncSetAttribute(lstm_fwd_tc_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, FWD_SMEM));
  LFMQ_CUDA_CHECK(cudaFuncSetAttribute(lstm_fwd_tc_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, FWD_SMEM));
  // how many 4-CTA clusters can be co-resident (one CTA per SM because of shared memory)
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = dim3(TC_NC * (m.n_sms / TC_NC));
  cfg.blockDim = dim3(FWD_THREADS);
  cfg.dynamicSmemBytes = FWD_SMEM;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeClusterDimension;
  attr[0].val.clusterDim.x = TC_NC;
  attr[0].val.clusterDim.y = 1;
  attr[0].val.clusterDim.z = 1;
  cfg.attrs = attr;
  cfg.numAttrs = 1;
  int nclusters = 0;
  LFMQ_CUDA_CHECK(cudaOccupancyMaxActiveClusters(&nclusters, lstm_fwd_tc_kernel<true>, &cfg));
  if (nclusters < 1) {
    LFMQ_SET_ERR("no 4-CTA cluster of the forward kernel fits on this device");
    return LFMQ_ERR_UNSUPPORTED;
  }
  m.max_clusters = nclusters;
  m.enabled = true;
  st.weights_dirty = 1;
  return 0;
}

void tc_destroy(TcState& st) {
  delete st.impl;
  st.impl = nullptr;
}

static int tc_pack_weights(TcState& st, const float* params, cudaStream_t s) {
  TcImpl& m = *st.impl;
  if (!st.weights_dirty) return 0;
  const int nblk = (int)(((long)4 * TC_H * TC_H + 255) / 256);
  PackArgs a;
  a.I = m.I; a.O = m.O; a.eps = m.eps;
  a.nb_w = nblk;
  a.nb_h = (TC_H * 32 + 255) / 256;
  a.nb_u = m.train ? nblk : 0;      // K-slices of U for the backward recurrence
  a.W = params + m.oW; a.U = params + m.oU; a.bias = params + m.ob;
  a.Wo = params + m.oWo; a.bo = params + m.obo; a.gamma = params + m.ogamma; a.beta = params + m.obeta;
  a.mean = params + m.omean; a.var = params + m.ovar;
  a.Up = m.Up; a.Wp = m.Wp; a.Ubk = m.Ubk; a.WoTp = m.WoTp; a.WoSp = m.WoSp; a.biasp = m.biasp; a.bop = m.bop;
  if (int rc = launch_pdl(pack_all_kernel, dim3(a.nb_w + a.nb_h + a.nb_u), dim3(256), 0, s, 1, true, a)) return rc;
  st.weights_dirty = 0;
  return 0;
}

static int tc_run_recurrence(TcState& st, const float* x, int B, bool save, cudaStream_t s) {
  TcImpl& m = *st.impl;
  const long bt = (long)B * m.T * 5;
  if (int rc = launch_pdl(xh_fill_x_kernel, dim3((int)((bt + 255) / 256)), dim3(256), 0, s, 1, true, B, m.T, m.I, x, m.xh)) return rc;
  const int n_tiles = (B + 127) / 128;
  FwdParams p;
  p.B = B; p.T = m.T;
  p.n_clusters = n_tiles < m.max_clusters ? n_tiles : m.max_clusters;
  p.n_iters = (n_tiles + p.n_clusters - 1) / p.n_clusters;
  p.n_tiles = n_tiles;
  p.k16_x = (m.I + 15) / 16;
  p.n_tiles_cap = (m.maxB + 127) / 128;
  p.xh = m.xh;
  p.gates = save ? m.gates : nullptr;
  p.cst = save ? m.cst : nullptr;
  p.biasp = m.biasp;
  if (save) {
    if (int rc = launch_pdl(lstm_fwd_tc_kernel<true>, dim3(TC_NC * p.n_clusters), dim3(FWD_THREADS), FWD_SMEM, s, TC_NC, true, p,
                            m.tm_h, m.tm_x, m.tm_u, m.tm_w))
      return rc;
  } else {
    if (int rc = launch_pdl(lstm_fwd_tc_kernel<false>, dim3(TC_NC * p.n_clusters), dim3(FWD_THREADS), FWD_SMEM, s, TC_NC, true, p,
                            m.tm_h, m.tm_x, m.tm_u, m.tm_w))
      return rc;
  }
  return 0;
}

static int tc_run_head(TcState& st, const lfmq_config& c, const float* params, float* grads, const float* y, int B,
                       int64_t row0, int64_t step, const float* denom, float* preds, float* out2, bool train,
                       cudaStream_t s) {
  TcImpl& m = *st.impl;
  HeadParams h;
  h.B = B; h.T = m.T; h.O = m.O; h.target_idx = c.target_idx; h.train = train ? 1 : 0;
  h.xh = m.xh;
  h.gamma = params + m.ogamma; h.beta = params + m.obeta; h.mean = params + m.omean; h.var = params + m.ovar;
  h.eps = c.bn_epsilon;
  h.Wo = params + m.oWo; h.bo = params + m.obo;
  h.y = y; h.denom = denom; h.p1 = c.target_lambda; h.p2 = c.rnn_lambda;
  h.use_dropout = (c.train && c.dropout > 0.f) ? 1 : 0;
  h.key = dropout_key(c.seed, 0, step, c.dropout);
  h.row0 = row0;
  h.preds = preds;
  // dhout / fp32 dpred are only produced on the dropout (SIMT) path; the tensor-core head leaves bf16 dpred tiles (dpb)
  const bool simt_train = train && c.train && c.dropout > 0.f;
  h.dhout = simt_train ? m.dhout : nullptr;
  h.dpred = simt_train ? m.dpred : nullptr;
  h.partial = m.head_part;
  const int n_btiles = (B + 127) / 128;
  const int n_tiles_cap = (m.maxB + 127) / 128;
  int grid = m.T * n_btiles;
  if (grid > m.head_ctas) grid = m.head_ctas;
  h.partial = m.head_part;
  HeadTcWeights hw;
  hw.WoTp = m.WoTp; hw.bop = m.bop;
  const bool use_tc = !h.use_dropout;       // the BN fold into the head weights needs y = a*h + b
  int n_wcta = m.head_wctas;
  if (train) {
    if (use_tc) {
      if (int rc = launch_pdl(head_tc_kernel<true>, dim3(grid), dim3(HT_THREADS), HT_SMEM, s, 1, true, h, hw, m.tm_h128, m.tm_wot,
                              m.tm_dpb, n_btiles, n_tiles_cap, m.head_wpart))
        return rc;
      n_wcta = grid;
    } else {
      head_rows_kernel<true><<<grid, 128, HROWS_SMEM, s>>>(h, m.tm_h128, n_btiles, n_tiles_cap);
      LFMQ_LAUNCH_CHECK();
      head_wgrad_kernel<<<m.head_wctas, 256, 0, s>>>(h, m.head_wpart);
      LFMQ_LAUNCH_CHECK();
    }
  } else {
    if (use_tc) {
      if (int rc = launch_pdl(head_tc_kernel<false>, dim3(grid), dim3(HT_THREADS), HT_SMEM, s, 1, true, h, hw, m.tm_h128,
                              m.tm_wot, m.tm_wot, n_btiles, n_tiles_cap, (float*)nullptr))
        return rc;
    } else {
      head_rows_kernel<false><<<grid, 128, HROWS_SMEM, s>>>(h, m.tm_h128, n_btiles, n_tiles_cap);
      LFMQ_LAUNCH_CHECK();
    }
  }
  if (y) {
    const int n_out = HWG_PART + HEAD_PART;
    if (int rc = launch_pdl(head_reduce_kernel, dim3((n_out * 32 + 255) / 256), dim3(256), 0, s, 1, true, grid,
                            (const float*)m.head_part, n_wcta, (const float*)m.head_wpart, m.O, B, denom, c.target_lambda,
                            c.rnn_lambda, train ? 1 : 0, grads ? grads + m.oWo : (float*)nullptr,
                            grads ? grads + m.obo : (float*)nullptr, grads ? grads + m.ogamma : (float*)nullptr,
                            grads ? grads + m.obeta : (float*)nullptr, out2))
      return rc;
    if (train && use_tc) {
      if (int rc = launch_pdl(head_fold_kernel, dim3((TC_H + 127) / 128), dim3(128), 0, s, 1, true, m.O, grads + m.oWo,
                              (const float*)(grads + m.obo), grads + m.ogamma, grads + m.obeta, params + m.oWo,
                              params + m.ogamma, params + m.obeta, params + m.omean, params + m.ovar, c.bn_epsilon))
        return rc;
    }
  }
  return 0;
}

int tc_forward(TcState& st, const lfmq_config& c, const float* params, const float* x, int B, int64_t row0,
               int64_t step, float* preds, bool save, cudaStream_t s) {
  if (!st.impl || !st.impl->enabled) {
    LFMQ_SET_ERR("bf16 path not initialised");
    return LFMQ_ERR_UNSUPPORTED;
  }
  int rc;
  if ((rc = tc_pack_weights(st, params, s))) return rc;
  st.prof->begin(LFMQ_REGION_FWD, s);
  if ((rc = tc_run_recurrence(st, x, B, save, s))) return rc;
  st.prof->end(LFMQ_REGION_FWD, s);
  if (preds) {
    st.prof->begin(LFMQ_REGION_HEAD, s);
    if ((rc = tc_run_head(st, c, params, nullptr, nullptr, B, row0, step, nullptr, preds, nullptr, false, s))) return rc;
    st.prof->end(LFMQ_REGION_HEAD, s);
  }
  return 0;
}

int tc_backward_impl(TcState& st, const lfmq_config& c, const float* params, float* grads, int B, bool fused,
                     cudaStream_t s);

int tc_backward(TcState& st, const lfmq_config& c, const float* params, float* grads, const float* x, const float* y,
                int B, int64_t row0, int64_t step, const float* denom, float* tail, cudaStream_t s) {
  if (!st.impl || !st.impl->enabled) {
    LFMQ_SET_ERR("bf16 path not initialised");
    return LFMQ_ERR_UNSUPPORTED;
  }
  int rc;
  if ((rc = tc_pack_weights(st, params, s))) return rc;
  st.prof->begin(LFMQ_REGION_FWD, s);
  if ((rc = tc_run_recurrence(st, x, B, true, s))) return rc;
  st.prof->end(LFMQ_REGION_FWD, s);
  st.prof->begin(LFMQ_REGION_HEAD, s);
  if ((rc = tc_run_head(st, c, params, grads, y, B, row0, step, denom, nullptr, tail, true, s))) return rc;
  st.prof->end(LFMQ_REGION_HEAD, s);
  // the tensor-core head (no dropout) leaves dLoss/dpred tiles for the backward kernel to expand on its own MMAs
  return tc_backward_impl(st, c, params, grads, B, /*fused=*/!(c.train && c.dropout > 0.f), s);
}

}  // namespace lfmq

// =============================================================================================
// Persistent backward recurrence (reverse t inside the kernel), clusters of 4 CTAs per 128-row tile.
//   CTA r owns hidden units [64r, 64r+64): it computes dz_t for its 256 gate columns (pointwise, SURVEY App. A.4),
//   stages them as the A operand in shared memory and multiplies by ITS K-slice of U (resident for the whole unroll):
//       partial_r[128 x 256] = dz_t[:, own 256 gate cols] * U[all 256 hidden, own gate cols]^T       (wgmma)
//   dh_{t-1}[:, slice q] = sum_r partial_r[:, slice q]: each CTA writes the three foreign 128x64 slices, as bf16,
//   straight into the owners' shared memory (st.async through distributed shared memory) -- a reduce-scatter whose
//   volume (48 KB in per CTA and step) is 5x smaller than all-gathering dz.
//   K order inside the slice: k' = 64*jb + 16*g + jj  <->  gate column g*H + 64r + 16*jb + jj, so hidden chunk jb
//   (16 units x 4 gates) is one 64-wide k-block and its MMAs overlap the pointwise work of chunk jb+1.
//   The N order of the resident U slice is rotated per CTA: accumulator columns 64d .. 64d+63 are hidden slice
//   (r + d) mod 4, so the CTA's own slice is always columns 0..63.
// =============================================================================================
namespace lfmq {

struct BwdParams {
  int B, T, n_iters, n_clusters, n_tiles, n_tiles_cap;
  const __nv_bfloat16* gates;
  const __nv_bfloat16* cst;
  const __nv_bfloat16* dhout;
};

constexpr int BWD_NC = 4;
// Warpgroups 0 and 1: pointwise gate gradients, A-operand staging, MMAs and partial exchange for rows 0-63 / 64-127 of
// the tile (the accumulator lives in their registers); warpgroup 2: warp 8 = TMA producer.  setmaxnreg moves the
// registers of the producer warpgroup to the two that hold 128 accumulators each.
constexpr int BWD_THREADS = 384;
constexpr int BWD_W_PROD = 8;
constexpr uint32_t SB_U = 0;                    // 4 k-blocks x [256 x 128 B]
constexpr uint32_t SB_A = 131072;               // 2 stages x [128 x 128 B]
constexpr uint32_t SB_R = 163840;               // received partial slices [slot d-1][chunk jb][consumer thread][16 B]
constexpr uint32_t SB_DPB = 212992;             // FUSED: dLoss/dpred tile of one step [128 x 64 B], SW64
constexpr uint32_t SB_WOS = 221184;             // FUSED: (Wo gamma inv) rows of this CTA's 64 hidden units [64 x 64 B], SW64
constexpr uint32_t SB_BARS = 225280;
constexpr uint32_t BWD_SMEM = SB_BARS + 256 + 1024;

struct BwdBars {
  uint64_t w_full;
  uint64_t recv_full[2];         // per consumer warpgroup: the peers' partial slices for its 64 rows have landed
  uint64_t slot_free[2];         // per consumer warpgroup: the peers have read the slices this CTA last sent them
  uint64_t dpb_full, dpb_free;   // FUSED: the dpred tile has landed / the MMAs reading it have completed
};

__device__ __forceinline__ uint32_t ld_b32(const __nv_bfloat16* p) { return *reinterpret_cast<const uint32_t*>(p); }

// FUSED (no dropout in the head): dLoss/dh of the head is not read from HBM.  With dy = dpred Wo^T it equals
// dpred (Wo gamma inv)^T; each warpgroup adds that product for this CTA's 64 hidden units (M64 x N64 x K32 on the 8 KB
// dpred tile) into the own-slice columns of its accumulator.
template <bool FUSED>
__global__ void __launch_bounds__(BWD_THREADS, 1)
    lstm_bwd_tc_kernel(BwdParams p, const __grid_constant__ CUtensorMap tm_ubk, const __grid_constant__ CUtensorMap tm_dzst,
                       const __grid_constant__ CUtensorMap tm_dpb, const __grid_constant__ CUtensorMap tm_wos) {
  extern __shared__ uint8_t smem_raw[];
  // Aligned by an offset from smem_raw rather than by masking a generic address, so that the compiler still knows the
  // pointer is shared: the staging stores and slice reads below then take 32-bit shared addresses (STS / LDS), not
  // 64-bit generic ones, which would be hoisted out of the step loop and held in registers.
  uint8_t* smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);
  BwdBars* bars = reinterpret_cast<BwdBars*>(smem + SB_BARS);
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const uint32_t rank = cluster_ctarank();
  const int cid = blockIdx.x / BWD_NC;
  const int T = p.T;

  if (tid == 0) {
    mbar_init(&bars->w_full, 1);
    for (int i = 0; i < 2; ++i) {
      mbar_init(&bars->recv_full[i], 1);
      mbar_init(&bars->slot_free[i], BWD_NC - 1);   // one arrive per peer
    }
    mbar_init(&bars->dpb_full, 1);
    mbar_init(&bars->dpb_free, 8);          // one arrive per consumer warp
    fence_mbar_init();
  }
  __syncthreads();
  cluster_sync_all();
  // programmatic dependent launch: the weight slices (packed at the start of the step) load under the predecessor's tail
  if (!(warp == BWD_W_PROD && lane == 0)) pdl_sync();

  if (warp >= 8) {
    setmaxnreg_dec<24>();
    if (warp == BWD_W_PROD && lane == 0) {
      // ===================== TMA producer: weights once, then (FUSED) the dpred tile of every step =========
      mbar_arrive_expect_tx(&bars->w_full, 131072 + (FUSED ? 4096 : 0));
      for (int jb = 0; jb < 4; ++jb)
        for (int d = 0; d < 4; ++d)
          tma_load_2d(smem + SB_U + jb * 32768 + d * 8192, &tm_ubk, &bars->w_full, jb * 64,
                      (int)rank * 256 + (int)((rank + d) & 3) * 64);
      if (FUSED) tma_load_2d(smem + SB_WOS, &tm_wos, &bars->w_full, 0, rank * 64);
      pdl_sync();
      if (FUSED) {
        uint32_t n_dp = 0;
        for (int it = 0; it < p.n_iters; ++it) {
          const int tile = it * p.n_clusters + cid;
          if (tile >= p.n_tiles) break;                   // clusters without a tile in the last round
          // dpred tile of time step td into the single staging buffer, once the MMAs that read the previous one are done
          for (int td = T - 1; td >= 0; --td) {
            if (n_dp > 0) mbar_wait(&bars->dpb_free, (n_dp - 1) & 1);
            ++n_dp;
            mbar_arrive_expect_tx(&bars->dpb_full, 8192);
            tma_load_2d(smem + SB_DPB, &tm_dpb, &bars->dpb_full, 0, (td * p.n_tiles_cap + tile) * 128);
          }
        }
      }
    }
  } else {
    setmaxnreg_inc<240>();
    // ===================== consumers =====================
    // Warpgroup wg owns rows 64 wg .. 64 wg + 63.  Accumulator fragment (m64 x n256): register i holds row
    // r0 + 8 ((i >> 1) & 1), column 8 (i >> 2) + 2 cq + (i & 1).  Own slice = registers 0..31: unit 16 jb + jj of this
    // CTA's 64, jj = 8 q + 2 cq + e, is register 4 (2 jb + q) + 2 h + e.
    // Register budget: 128 accumulators, 32 dc, 24 rown and 24 operand words per thread leave about 30 of the 240
    // registers for everything else.  So wg comes through a shuffle from lane 0, which ptxas knows to be warp-uniform:
    // the MMAs are issued from one branch per warpgroup (uniform, so the wgmma pipeline is not serialised) with
    // descriptors formed in uniform registers from the shared-memory base, not held per thread across the step loop.
    const int wg = __shfl_sync(0xffffffffu, warp >> 2, 0), w = warp & 3, cq = lane & 3;
    const int r0 = 64 * wg + 16 * w + (lane >> 2);
    const bool elected = (tid & 127) == 0;
    const uint32_t wg_bar = 2 + wg;
    // this thread's word of row r0 in a staged A operand, 16-byte chunk 0 of the SW128 pattern: chunk k lies at
    // st_off ^ (k << 4), since the stage is 1024-byte aligned and row r0 (and r0 + 8) swizzles by r0 & 7
    const uint32_t st_off = r0 * 128 + ((r0 & 7) << 4) + 4 * cq;
    // Received partials, in fragment order: thread i of the sending CTA holds in acc[32 d .. 32 d + 31] (d = (dst - src)
    // mod 4) exactly the rows and columns that thread i here adds to acc[0..31].  Slot d - 1 holds the slice of peer
    // (rank + d) mod 4 as [chunk jb][consumer thread][4 words]: vector jb of a thread is the four packed bf16x2 words
    // of chunk jb, word 2 h + q (registers 8 jb + 2 h + 4 q).  The sender writes it with one 16-byte st.async, a warp
    // covering 512 contiguous bytes; it is read back as two 8-byte halves, one per row half h (three live 16-byte
    // vectors would spill).
    const uint32_t recv_off = SB_R + tid * 16;
    const long tstride = (long)p.n_tiles_cap * 8 * 4 * 2 * 32 * 16;   // cst elements per time step
    float acc[128];
    // dLoss/dh (recurrent + head part) of the own slice for the current step: chunk 0's eight values are read straight
    // from acc[0..7] (nothing overwrites them before chunk 0's MMAs), chunks 1-3 are copied out, rown[i] = acc[8 + i]
    float rown[24];
    float dc[32];                            // carried dLoss/dc, indexed like acc[0..31]
    // exchanges sent so far: step t sends the partials that the peers' step t - 1 receives, so the receive waited for at
    // step t is the (n_ex - 1)-th phase of recv_full, and the send waits for the n_ex-th phase of slot_free
    uint32_t n_ex = 0, n_dpf = 0;
    mbar_wait(&bars->w_full, 0);

    // head part of dLoss/dh (dpred (Wo gamma inv)^T) into the own-slice registers: accumulate = 0 at a tile's first step
    auto dy_mma = [&](uint32_t accumulate) {
      mbar_wait(&bars->dpb_full, (n_dpf++) & 1);
      wgmma_fence();
      auto mma = [&](const uint8_t* a_tile) {
#pragma unroll
        for (int k16 = 0; k16 < 2; ++k16) {
          const uint64_t da = make_smem_desc(smem_u32(a_tile) + k16 * 32, 0, 512, LAYOUT_SW64);
          const uint64_t db = make_smem_desc(smem_u32(smem + SB_WOS) + k16 * 32, 0, 512, LAYOUT_SW64);
          wgmma_m64n64k16<0, 0>(*reinterpret_cast<float(*)[32]>(acc), da, db, (accumulate || k16 > 0) ? 1u : 0u);
        }
      };
      if (wg == 0) mma(smem + SB_DPB);
      else mma(smem + SB_DPB + 4096);
      wgmma_commit();
    };

    for (int it = 0; it < p.n_iters; ++it) {
      const int tile = it * p.n_clusters + cid;
      if (tile >= p.n_tiles) break;
#pragma unroll
      for (int i = 0; i < 32; ++i) dc[i] = 0.f;
      if (FUSED) {                             // the head's dLoss/dh_{T-1}: nothing recurrent to add to yet
        dy_mma(0);
        wgmma_wait<0>();
        fence_regs(acc);
        if (lane == 0) mbar_arrive(&bars->dpb_free);
#pragma unroll
        for (int i = 0; i < 24; ++i) rown[i] = acc[8 + i];
      } else {
#pragma unroll
        for (int i = 0; i < 8; ++i) acc[i] = 0.f;
#pragma unroll
        for (int i = 0; i < 24; ++i) rown[i] = 0.f;
      }
      for (int t = T - 1; t >= 0; --t) {
        const bool has_rec = t < T - 1;
        // This thread's first element of the step's saved state and head dLoss/dh (row r0, units 2 cq, 2 cq + 1 of
        // chunk 0).  Rows r0 and r0 + 8 lie in the same 32-row quadrant, so every (chunk, h, q, gate) operand is a
        // constant offset from these three pointers: no per-operand address arithmetic is live across the chunk loop.
        const long sblk = (((long)t * p.n_tiles_cap + tile) * 8 + 2 * rank) * 4 + (r0 >> 5);
        const __nv_bfloat16* gbase = p.gates + sblk * 4096 + (r0 & 31) * 16 + 2 * cq;
        const __nv_bfloat16* cbase = p.cst + sblk * 1024 + (r0 & 31) * 16 + 2 * cq;
        const __nv_bfloat16* dbase =
            p.dhout + ((((long)t * p.n_tiles_cap + tile) * 4 + rank) * 4 + (r0 >> 5)) * 2048 + (r0 & 31) * 16 + 2 * cq;
        // Saved-state operands of one chunk, all requested before the first is used: one memory latency per chunk.
        // They do not depend on the exchange, so chunk 0's go out before the wait for the peers' partials, and chunk
        // jb + 1's right after chunk jb's staging stores, into the registers chunk jb no longer needs.
        uint32_t gi[2][2], gf[2][2], gg[2][2], go[2][2], ct[2][2], cp[2][2], dhp[2][2];     // [h][q]
        auto load_chunk = [&](int jb) {
#pragma unroll
          for (int h = 0; h < 2; ++h) {
            const bool valid = (long)tile * 128 + r0 + 8 * h < p.B;
#pragma unroll
            for (int q = 0; q < 2; ++q) {
              if (valid) {
                const int so = (jb >> 1) * 4 * 4096 + (jb & 1) * 512 + 128 * h + 8 * q;   // gates; cst: the same / 4
                const int co = (jb >> 1) * 4 * 1024 + (jb & 1) * 512 + 128 * h + 8 * q;
                gi[h][q] = ld_b32(gbase + so);
                gf[h][q] = ld_b32(gbase + so + 1024);
                gg[h][q] = ld_b32(gbase + so + 2048);
                go[h][q] = ld_b32(gbase + so + 3072);
                ct[h][q] = ld_b32(cbase + co);
                cp[h][q] = t > 0 ? ld_b32(cbase + co - tstride) : 0u;
                dhp[h][q] = FUSED ? 0u : ld_b32(dbase + jb * 512 + 128 * h + 8 * q);
              } else {
                gi[h][q] = gf[h][q] = gg[h][q] = go[h][q] = ct[h][q] = cp[h][q] = dhp[h][q] = 0u;
              }
            }
          }
        };
        load_chunk(0);
        if (has_rec) mbar_wait_cluster(&bars->recv_full[wg], (n_ex + 1) & 1);
#pragma unroll
        for (int jb = 0; jb < 4; ++jb) {
          const int st = jb & 1;
          uint8_t* stage = smem + SB_A + st * 16384;
          // the stage is free: the MMAs of its previous use (two chunks ago) and the dz store that read it are done
          wgmma_wait<1>();
          if (elected) bulk_wait_group_read1();
          named_bar_sync(wg_bar, 128);
#pragma unroll
          for (int h = 0; h < 2; ++h) {
            // dLoss/dh of the own slice: own part, plus the peers' slices d = 1, 2, 3 in that order, summed in place
            // (acc[0..7] are rewritten by chunk 0's MMAs, rown[] by the next step)
            auto own = [&](int ri) -> float& { return jb == 0 ? acc[ri] : rown[ri - 8]; };
            if (has_rec) {
#pragma unroll
              for (int d = 0; d < 3; ++d) {
                const uint2 v = *reinterpret_cast<const uint2*>(smem + recv_off + d * 16384 + jb * 4096 + 8 * h);
                const int ri = 8 * jb + 2 * h;
                own(ri) += bf16_lo(v.x);
                own(ri + 1) += bf16_hi(v.x);
                own(ri + 4) += bf16_lo(v.y);
                own(ri + 5) += bf16_hi(v.y);
              }
            }
#pragma unroll
            for (int q = 0; q < 2; ++q) {
              const int ri = 4 * (2 * jb + q) + 2 * h;       // register of (unit jj, e = 0) in acc[0..31] / dc
              const float rec0 = own(ri), rec1 = own(ri + 1);
              // gate-gradient algebra in packed bf16x2 (two units per word); only the carried dLoss/dc stays in fp32
              // registers.  SURVEY App. A.4.
              const uint32_t i2 = gi[h][q], f2 = gf[h][q], g2 = gg[h][q], o2 = go[h][q];
              const uint32_t dh2 = FUSED ? pack_bf16x2(rec0, rec1) : add_bf16x2(dhp[h][q], pack_bf16x2(rec0, rec1));
              const uint32_t tc2 = tanh_bf16x2(ct[h][q]);
              const uint32_t omtc2 = fma_bf16x2(neg_bf16x2(tc2), tc2, BF16X2_ONE);        // 1 - tanh(c)^2
              const uint32_t t1 = mul_bf16x2(mul_bf16x2(dh2, o2), omtc2);                 // dh * o * (1 - tc^2)
              const float dcn0 = dc[ri] + bf16_lo(t1);
              const float dcn1 = dc[ri + 1] + bf16_hi(t1);
              dc[ri] = dcn0 * bf16_lo(f2);
              dc[ri + 1] = dcn1 * bf16_hi(f2);
              const uint32_t dcn2 = pack_bf16x2(dcn0, dcn1);
              const uint32_t omi = fma_bf16x2(neg_bf16x2(i2), i2, i2);                    // i (1 - i)
              const uint32_t omf = fma_bf16x2(neg_bf16x2(f2), f2, f2);                    // f (1 - f)
              const uint32_t omg = fma_bf16x2(neg_bf16x2(g2), g2, BF16X2_ONE);            // 1 - g^2
              const uint32_t omo = fma_bf16x2(neg_bf16x2(o2), o2, o2);                    // o (1 - o)
              const uint32_t z[4] = {mul_bf16x2(dcn2, mul_bf16x2(g2, omi)), mul_bf16x2(dcn2, mul_bf16x2(cp[h][q], omf)),
                                     mul_bf16x2(dcn2, mul_bf16x2(i2, omg)), mul_bf16x2(mul_bf16x2(dh2, tc2), omo)};
              // A operand k-block jb: row m, 16-byte chunk 2g+q holds gate g, units 8q..8q+7 (SW128 K-major)
#pragma unroll
              for (int g = 0; g < 4; ++g)
                *reinterpret_cast<uint32_t*>(stage + 1024 * h + (st_off ^ ((2 * g + q) << 4))) = z[g];
            }
          }
          if (jb < 3) load_chunk(jb + 1);
          fence_proxy_async_smem();
          named_bar_sync(wg_bar, 128);
          wgmma_fence();
          auto chunk_mma = [&](const uint8_t* a_tile) {     // one branch per warpgroup, see wg above
#pragma unroll
            for (int k16 = 0; k16 < 4; ++k16) {
              const uint64_t da = make_smem_desc(smem_u32(a_tile) + k16 * 32, 0, 1024, LAYOUT_SW128);
              const uint64_t db = make_smem_desc(smem_u32(smem + SB_U + jb * 32768) + k16 * 32, 0, 1024, LAYOUT_SW128);
              wgmma_m64n256k16<0, 0>(acc, da, db, (jb | k16) != 0);
            }
          };
          if (wg == 0) chunk_mma(stage);
          else chunk_mma(stage + 8192);
          wgmma_commit();
          // dz_t of the chunk leaves for HBM straight from the A operand: one TMA store per warpgroup (64 rows x 128 B,
          // rows >= B clipped).  dz keeps the operand's column order [16-unit block][gate][16] (see tc_layout);
          // wgrad_reduce_kernel puts the gate columns back in order.
          if (elected) {
            tma_store_3d(&tm_dzst, stage + wg * 8192, (4 * (int)rank + jb) * 64, t, tile * 128 + 64 * wg);
            bulk_commit_group();
          }
        }
        // The warpgroup has read its received slices of this step (chunk 3's second barrier follows the last reads):
        // arm recv_full for step t - 1, then tell the peers their slots are free.  The arm precedes the arrive that
        // lets any peer send, so no tx completes on a phase before it is armed.
        if (elected && t > 0) {
          mbar_arrive_expect_tx(&bars->recv_full[wg], (BWD_NC - 1) * 8192);
#pragma unroll
          for (uint32_t d = 1; d < BWD_NC; ++d) mbar_arrive_cluster(mapa_u32(smem_u32(&bars->slot_free[wg]), (rank + d) & 3));
        }
        if (FUSED && t > 0) dy_mma(1);         // head part of dLoss/dh_{t-1}, read (acc[0..7], rown) next step
        wgmma_wait<0>();
        fence_regs(acc);
        if (FUSED && t > 0 && lane == 0) mbar_arrive(&bars->dpb_free);
        if (t > 0) {
          // ---- export the foreign slices of partial_t (needed by the peers for step t-1) into their shared memory ----
          // Peer (rank + d) mod 4 files this CTA's slice in its slot 3 - d.  Its warpgroup wg has read what this CTA
          // sent last step once slot_free[wg] completes; the stores complete tx on its recv_full[wg].
          mbar_wait_cluster(&bars->slot_free[wg], (n_ex++) & 1);
#pragma unroll
          for (int d = 1; d < BWD_NC; ++d) {
            const uint32_t peer = (rank + (uint32_t)d) & 3;
            const uint32_t dst = mapa_u32(smem_u32(smem + recv_off + (3 - d) * 16384), peer);
            const uint32_t bar = mapa_u32(smem_u32(&bars->recv_full[wg]), peer);
#pragma unroll
            for (int jb = 0; jb < 4; ++jb) {
              const int i = 32 * d + 8 * jb;
              st_async_v4(dst + jb * 4096,
                          make_uint4(pack_bf16x2(acc[i], acc[i + 1]), pack_bf16x2(acc[i + 4], acc[i + 5]),
                                     pack_bf16x2(acc[i + 2], acc[i + 3]), pack_bf16x2(acc[i + 6], acc[i + 7])),
                          bar);
            }
          }
#pragma unroll
          for (int i = 0; i < 24; ++i) rown[i] = acc[8 + i];
        }
      }
    }
    if (elected) bulk_wait_group0();            // all dz stores complete before the kernel ends
  }
  __syncwarp();
  cluster_sync_all();          // nobody leaves while peers may still store into / arrive on this CTA
}

// =============================================================================================
// Weight gradients as ONE wgmma GEMM over all B*(T+1) rows (wgrad_gemm):  D[384 x 1024] = xh^T * dz   (both MN-major)
//   rows 0..255 -> dU, rows 256..256+I-1 -> dW, row 288 (the constant-one column) -> db.
// =============================================================================================
// Sums the K-split partials and scatters D rows into dU / dW / db of the flat gradient vector.  D's columns are in
// dz's order [16-unit block][gate][16]; the gradients want gate-major columns g*H + unit.
__global__ void wgrad_reduce_kernel(int S, int I, const float* __restrict__ partial, float* __restrict__ gU,
                                    float* __restrict__ gW, float* __restrict__ gb) {
  pdl_sync();
  const long idx = (long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= (long)384 * 1024) return;
  const int row = (int)(idx / 1024), np = (int)(idx % 1024);
  const int n = ((np % 64) / 16) * TC_H + (np / 64) * 16 + (np % 16);
  float* dst = nullptr;
  if (row < TC_H) dst = gU + (long)row * 1024 + n;
  else if (row < TC_H + I) dst = gW + (long)(row - TC_H) * 1024 + n;
  else if (row == TC_ONE) dst = gb + n;
  if (!dst) return;
  float s = 0.f;
  for (int z = 0; z < S; ++z) s += partial[(long)z * 384 * 1024 + idx];
  *dst = s;
}

int tc_backward_impl(TcState& st, const lfmq_config& c, const float* params, float* grads, int B, bool fused,
                     cudaStream_t s) {
  TcImpl& m = *st.impl;
  int rc;
  if (!m.bwd_ready) {
    LFMQ_CUDA_CHECK(cudaFuncSetAttribute(lstm_bwd_tc_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, BWD_SMEM));
    LFMQ_CUDA_CHECK(cudaFuncSetAttribute(lstm_bwd_tc_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, BWD_SMEM));
    if ((rc = wgrad_gemm_init())) return rc;
    // boxes of 64 hidden units: the kernel loads its K-slice of U in rotated N order (own hidden slice first)
    if ((rc = encode_map_2d(&m.tm_ubk, m.Ubk, 256, 4 * TC_H, 512, 64, 64, CU_TENSOR_MAP_SWIZZLE_128B))) return rc;
    cudaLaunchConfig_t qc = {};
    qc.gridDim = dim3(BWD_NC * (m.n_sms / BWD_NC));
    qc.blockDim = dim3(BWD_THREADS);
    qc.dynamicSmemBytes = BWD_SMEM;
    cudaLaunchAttribute qa[1];
    qa[0].id = cudaLaunchAttributeClusterDimension;
    qa[0].val.clusterDim.x = BWD_NC;
    qa[0].val.clusterDim.y = 1;
    qa[0].val.clusterDim.z = 1;
    qc.attrs = qa;
    qc.numAttrs = 1;
    int ncl = 0;
    LFMQ_CUDA_CHECK(cudaOccupancyMaxActiveClusters(&ncl, lstm_bwd_tc_kernel<true>, &qc));
    if (ncl < 1) {
      LFMQ_SET_ERR("no 4-CTA cluster of the backward kernel fits on this device");
      return LFMQ_ERR_UNSUPPORTED;
    }
    m.bwd_max_clusters = ncl;
    m.bwd_ready = true;
  }
  const size_t T = (size_t)m.T;
  st.prof->begin(LFMQ_REGION_BWD, s);
  {
    BwdParams bp;
    const int n_tiles = (B + 127) / 128;
    bp.B = B; bp.T = m.T;
    bp.n_tiles_cap = (m.maxB + 127) / 128;
    bp.n_clusters = n_tiles < m.bwd_max_clusters ? n_tiles : m.bwd_max_clusters;
    bp.n_iters = (n_tiles + bp.n_clusters - 1) / bp.n_clusters;
    bp.n_tiles = n_tiles;
    bp.gates = m.gates; bp.cst = m.cst; bp.dhout = m.dhout;
    // dz as [b][t][1024] with columns ordered [16-unit block][gate][16]: one warpgroup's part of a staged chunk =
    // 64 rows x 64 columns
    CUtensorMap tm_dzst;
    {
      const uint64_t dims[3] = {1024, (uint64_t)(T + 1), (uint64_t)B};
      const uint64_t strides[2] = {2048, (uint64_t)2048 * (T + 1)};
      const uint32_t box[3] = {64, 1, 64};
      if ((rc = encode_map_bf16(&tm_dzst, m.dz, 3, dims, strides, box, CU_TENSOR_MAP_SWIZZLE_128B))) return rc;
    }
    if (fused) {
      if ((rc = launch_pdl(lstm_bwd_tc_kernel<true>, dim3(BWD_NC * bp.n_clusters), dim3(BWD_THREADS), BWD_SMEM, s, BWD_NC, true, bp,
                           m.tm_ubk, tm_dzst, m.tm_dpb, m.tm_wos)))
        return rc;
    } else {
      if ((rc = launch_pdl(lstm_bwd_tc_kernel<false>, dim3(BWD_NC * bp.n_clusters), dim3(BWD_THREADS), BWD_SMEM, s, BWD_NC, true, bp,
                           m.tm_ubk, tm_dzst, m.tm_dpb, m.tm_wos)))
        return rc;
    }
  }
  st.prof->end(LFMQ_REGION_BWD, s);

  st.prof->begin(LFMQ_REGION_WGRAD, s);
  // MN-major maps over exactly the B*(T+1) rows of this call (rows beyond are zero-filled by TMA)
  const uint64_t rows = (uint64_t)B * (T + 1);
  CUtensorMap tm_a, tm_b;
  if ((rc = encode_map_2d(&tm_a, m.xh, TC_XH_LD, rows, TC_XH_LD * 2, 64, 64, CU_TENSOR_MAP_SWIZZLE_128B))) return rc;
  if ((rc = encode_map_2d(&tm_b, m.dz, 4 * TC_H, rows, 4 * TC_H * 2, 64, 64, CU_TENSOR_MAP_SWIZZLE_128B))) return rc;
  int S = 0, Mpad = 0;
  if ((rc = wgrad_gemm(tm_a, tm_b, (long)rows, TC_XH_LD, 4 * TC_H, m.wg_part, m.wg_part_elems, true, s, &S, &Mpad)))
    return rc;
  if ((rc = launch_pdl(wgrad_reduce_kernel, dim3((384 * 1024 + 255) / 256), dim3(256), 0, s, 1, true, S, m.I,
                       (const float*)m.wg_part, grads + m.oU, grads + m.oW, grads + m.ob)))
    return rc;
  st.prof->end(LFMQ_REGION_WGRAD, s);
  (void)params;
  (void)c;
  return 0;
}

}  // namespace lfmq
