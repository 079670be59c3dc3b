// General tensor-core path of the recurrent forecaster: every shape the H=256 / L=1 LSTM cluster kernels of lstm_tc.cu
// do not cover -- H a multiple of 64 up to 512, stacked layers, dropout and recurrent dropout (BASELINE configs[2]:
// H=512, L=2, dropout) -- and the fp32-tolerance mode LFMQ_PREC_BF16X3.  Training runs the LSTM point estimate;
// forward-only handles also run the GRU cell and the RNNUqRangeEstimate heads (MC dropout included).
//
// One wgmma tile-GEMM skeleton (TMA ring -> wgmma -> register accumulators -> epilogue in the same warpgroups) with
// these epilogues:
//   EPI_FWD    z_t = [h_{t-1} (*rec mask) | in_t] [U; W]   (one launch per time step and layer)
//              epilogue = bias, gate nonlinearities, c_t / h_t update, h_t -> next step's A operand, saved state
//   EPI_GRU_FWD  the same GEMM on the GRU's packed [U; W] (gate slots z | r | n_x | n_h, see gpack_kernel)
//              epilogue = Keras reset-after GRU update of h_t (carried in fp32), forward-only: nothing saved
//   EPI_HEAD_UQ  [pred | var pre-activation] = y [Wo | Wv] (N = 32), epilogue = biases, softplus floor
//   EPI_BWD    rec = dz_{t+1} U^T                           (one launch per time step and layer, reverse time)
//              epilogue = BPTT pointwise algebra of step t (SURVEY App. A.4) -> dz_t, carried dLoss/dc
//   EPI_STORE  C = A B^T as bf16 (dLoss/d(input) of layers above the first: dz W^T)
// Why launches per time step and not one persistent kernel here: [U; W] of H=512 is 2-4 MB in bf16 -- it fits neither one
// SM nor a portable cluster's shared memory next to the operand ring, so the weight tiles stream from L2 every step
// either way; with two CTAs per SM the epilogue of one tile overlaps the loads / MMAs of the other.  The H=256, L=1 case
// (weights resident in a 4-CTA cluster for the whole unroll) keeps its persistent kernels in lstm_tc.cu.
//
// Data layout (time-major, Bp = maxB rounded up to 128 rows, "blocked" = [..][row tile][16-unit block][piece][4 warps]
// [32 lanes][16] so that a warp's 32-byte-per-thread access is 1 KB contiguous):
//   hseq[l]  bf16 [T+1][Bp][H]    slot t = h_{t-1} (slot 0 zero): A operand of step t, input of BN/Dropout, A^T of dU
//   hmseq[l] bf16 [T+1][Bp][H]    recurrent dropout only: h_{t-1} * mask (what the recurrence and dU actually consume);
//                                 hmseq_lo[l] its low halves (bf16x3)
//   in[l]    bf16 [T][Bp][Ipad]   layer input (l = 0: x cast to bf16; l > 0: Dropout(BN(h_{l-1}))); in[L] feeds the head
//   gates[l] bf16 blocked [T][row tile][H/16][4 gates]   post-activation i, f, g, o;  cst[l] blocked [T][row tile][H/16]
//   dz       bf16 [T][Bp][4H]     gate pre-activation gradients, standard column order i|f|g|o (shared by the layers)
//   dy / dhout bf16 [T][Bp][H]    dLoss/dy_l (from the head or the layer above) and after Dropout/BN backward
#include "rnn_tc.h"

#include <cuda.h>
#include <cuda_bf16.h>
#include <stdlib.h>

#include <vector>

#include "kernels.h"
#include "sm90.cuh"

namespace lfmq {

using namespace sm90;

namespace {

// bf16 2-D map over a row-major [outer][inner] buffer, SWIZZLE_128B boxes of box_inner (= 64) x box_outer elements.
int gmap_2d(CUtensorMap* m, const void* base, uint64_t inner, uint64_t outer, uint32_t box_inner, uint32_t box_outer) {
  return encode_map_2d(m, base, inner, outer, inner * 2, box_inner, box_outer, CU_TENSOR_MAP_SWIZZLE_128B);
}

inline long cdivl(long a, long b) { return (a + b - 1) / b; }

}  // namespace

// =============================================================================================
// Tile GEMM skeleton
// =============================================================================================
// warps 0-7: two consumer warpgroups (MMAs + epilogue) per 128-row M tile, warp 8: TMA producer
constexpr int G_MAXSEG = 6;
constexpr int GBAR_N = 4096;       // step-barrier counters per handle: one per (persistent launch, row-tile group)

// One K segment: n_kb 64-wide k-blocks, A columns from a_col0 of map a_map, B columns from b_col0 of map b_map.
struct GSeg {
  int a_map, b_map, n_kb, a_col0, b_col0;
};
struct GArgs {
  int n_seg;
  GSeg seg[G_MAXSEG];
  int a_row_base;      // A row coordinate = a_row_base + 128 * (blockIdx.x + rt_off)
  int b_row_base;      // B row coordinate = b_row_base + BN * blockIdx.y
  int rt_off;          // first 128-row tile of this launch (the batch can be split over two concurrent launches)
  // Persistent mode (n_steps > 1): one launch runs n_steps consecutive time steps of a layer; step i works on A rows
  // a_row_base + i * row_step with EpiParams::t + i * t_step.  The A operand of a CTA's next step is written by the
  // gridDim.y CTAs of its own row-tile group (same blockIdx.x, all column tiles), so the steps are separated by one
  // barrier PER ROW-TILE GROUP (a counter in global memory; every CTA of the launch resident at once), not by a launch
  // boundary: CTA dispatch, barrier init and the wait for the whole previous grid to retire are paid
  // once, and the row-tile groups drift apart instead of hitting HBM in lockstep.
  int n_steps, row_step, t_step;
  int lin_cols;        // > 0: 1-D grid, CTA i = (row tile i / lin_cols, column tile i % lin_cols): the column tiles of a row
                       // tile are dispatched together and share its A tile in L2 (multi-wave GEMMs: EPI_STORE)
  unsigned int* gbar;  // [gridDim.x], zeroed before the launch; counts the group's CTAs that have finished a step
};

enum {   // _ACC: expf / tanhf (bf16x3)
  EPI_FWD = 0, EPI_BWD = 1, EPI_STORE = 2, EPI_FWD_ACC = 3, EPI_HEAD = 4, EPI_GRU_FWD = 5, EPI_GRU_FWD_ACC = 6,
  EPI_HEAD_UQ = 7
};
constexpr bool epi_is_fwd(int e) { return e == EPI_FWD || e == EPI_FWD_ACC || e == EPI_GRU_FWD || e == EPI_GRU_FWD_ACC; }
constexpr bool epi_is_head(int e) { return e == EPI_HEAD || e == EPI_HEAD_UQ; }

struct EpiParams {
  // common
  int t, T, B, Bp, H, NRT, NB16;
  int64_t row0;
  // forward
  const float* bias;            // [4H] in the packed column order (sigmoid gates pre-scaled by 1/2 unless accurate)
  float* cstate;                // fp32 blocked [row tile][H/16][4][32][16]: c_{t-1} in, c_t out (GRU: h_{t-1} in, h_t out)
  __nv_bfloat16* hseq;          // [T+1][Bp][H]
  __nv_bfloat16* hseq_lo;       // bf16x3: low halves of h
  __nv_bfloat16* hmseq;         // recurrent dropout: masked copy (null otherwise)
  __nv_bfloat16* gates;         // blocked, null: do not save
  __nv_bfloat16* cst;           // blocked, null: do not save
  int accurate;                 // 1: expf / tanhf (bf16x3 mode), 0: tanh.approx
  int use_rec;                  // recurrent dropout active
  DropoutKey rkey;
  // backward
  const __nv_bfloat16* dhout;   // [T][Bp][H]
  float* dcstate;               // fp32 blocked, carried dLoss/dc
  __nv_bfloat16* dz;            // [T][Bp][4H]
  int has_rec;                  // t < T-1: the accumulator holds dz_{t+1} U^T
  // store
  __nv_bfloat16* out;           // [rows][ldc]
  int ldc;
  // head (EPI_HEAD): pred = y Wo + bo, weighted MSE (losses.py:55-135), dLoss/dpred
  const float* hy;              // targets [B][T][O] fp32 or null
  const float* hdenom;          // {B_global, mask_count_global}
  const float* hrw;             // row weights of the training batch (nullable)
  const float* hbo;             // [O]
  float* hpreds;                // [B][T][O] fp32 or null
  __nv_bfloat16* hdpb;          // [T*Bp][64] bf16, cols >= 16 stay zero: dLoss/dpred rows (operand of the dy and dWo GEMMs)
  float* hpartial;              // [GH_PART][gridDim.x]
  float hp1, hp2;
  int hO, htarget, htrain;
  // forward, bf16x3 with recurrent dropout: low halves of the masked h
  __nv_bfloat16* hmseq_lo;
  // variance head (EPI_HEAD_UQ): var = max(softplus(y Wv + bv), 1e-6)
  const float* hbv;             // [O]
  float* hvar;                  // [B][T][O] fp32
};

// Two consumer warpgroups per CTA (rows 0-63 / 64-127 of the 128-row M tile, each with an m64 x BN accumulator in
// registers) and one TMA producer warp.  The forward (N = 256: 128 accumulator registers per thread) and backward
// steps run one CTA per SM; the multi-wave GEMMs (EPI_STORE, the heads) keep two CTAs per SM.  The ring takes whatever
// shared memory one / two resident CTAs leave: the loads are latency-bound, bytes in flight are what buys bandwidth.
template <int BN, int EPI>
struct GSmem {
  static constexpr uint32_t A_BYTES = 128 * 128;          // 128 rows x 64 bf16
  static constexpr uint32_t B_BYTES = BN * 128;
  static constexpr uint32_t STAGE = A_BYTES + B_BYTES;
  static constexpr int CTAS_PER_SM = (EPI == 2 || epi_is_head(EPI)) ? 2 : 1;      // (2 = EPI_STORE)
  static constexpr int NS = (int)((CTAS_PER_SM == 2 ? 98304u : 196608u) / STAGE);
  static constexpr uint32_t BARS = NS * STAGE;
  static constexpr uint32_t HEAD_ROWS = BARS + 256;        // heads: [128][BN + 1] fp32 accumulator rows
  static constexpr uint32_t TOTAL = HEAD_ROWS + (epi_is_head(EPI) ? 128 * (BN + 1) * 4 : 0) + 1024;   // + alignment slack
  static constexpr int THREADS = 2 * 128 + 32;
};

__device__ __forceinline__ float sigmoid_acc(float x) { return 1.0f / (1.0f + expf(-x)); }

// recurrent-dropout mask of the four units of quad j / 4 (the quad numbering of the SIMT path)
__device__ __forceinline__ void rec_mask4(const DropoutKey& k, int64_t grow, int H, int j, float m[4]) {
  dropout_quad(k, (uint64_t)grow * (uint64_t)(H / 4) + (uint64_t)(j / 4), m);
}

__device__ __forceinline__ uint32_t ld_b32(const __nv_bfloat16* p) { return *reinterpret_cast<const uint32_t*>(p); }
__device__ __forceinline__ void st_b32(__nv_bfloat16* p, uint32_t v) { *reinterpret_cast<uint32_t*>(p) = v; }

template <int BN>
__device__ __forceinline__ void wgmma_bn(float (&acc)[BN / 2], uint64_t da, uint64_t db, uint32_t accumulate) {
  if constexpr (BN == 256) wgmma_m64n256k16<0, 0>(acc, da, db, accumulate);
  if constexpr (BN == 128) wgmma_m64n128k16<0, 0>(acc, da, db, accumulate);
  if constexpr (BN == 64) wgmma_m64n64k16<0, 0>(acc, da, db, accumulate);
  if constexpr (BN == 32) wgmma_m64n32k16<0, 0>(acc, da, db, accumulate);
  if constexpr (BN == 16) wgmma_m64n16k16<0, 0>(acc, da, db, accumulate);
}

// Fragment coordinates of a consumer thread: rows m0 and m0 + 8 of the 128-row tile (register bit 1), columns
// 8 (i >> 2) + 2 cq + (i & 1).
struct Frag {
  int m0, cq;
};

// ---- EPI_FWD: gates, cell update, h_t (SURVEY App. A.1; rnn_point_estimate.py:80-87) ----------------------------
// Accumulator columns of a tile: [16-unit block][gate i|f|g|o][16] (the packed order of the B operand rows).  Gate g of
// unit jj = 8 q + 2 cq + e of block blk is register 32 blk + 4 (2 g + q) + 2 h + e.
template <bool ACC>
__device__ __forceinline__ void epi_fwd(const EpiParams& p, const float (&acc)[128], Frag f, int rt, int by,
                                        const float* bias_s) {
  constexpr int U = 64;                             // hidden units of this tile
  const int unit0 = by * U;
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    const int m = f.m0 + 8 * h;
    const long b = (long)rt * 128 + m;
    const bool valid = b < p.B;
#pragma unroll
    for (int blk = 0; blk < U / 16; ++blk) {
      const int gblk = (unit0 >> 4) + blk;
      float* cs = p.cstate + ((((long)rt * p.NB16 + gblk) * 4 + (m >> 5)) * 32 + (m & 31)) * 16;
      const float* bs = bias_s + blk * 64;        // this tile's packed bias, staged in shared memory (broadcast reads)
#pragma unroll
      for (int q = 0; q < 2; ++q) {
        const int jj = 8 * q + 2 * f.cq;
        const int j = unit0 + blk * 16 + jj;
        const float2 cprev = p.t > 0 ? *reinterpret_cast<const float2*>(cs + jj) : make_float2(0.f, 0.f);
        float gv[4][2], cn[2], hv[2];
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          const int ri = 32 * blk + 4 * q + 2 * h + e;
          const float zi = acc[ri] + bs[jj + e];
          const float zf = acc[ri + 8] + bs[16 + jj + e];
          const float zg = acc[ri + 16] + bs[32 + jj + e];
          const float zo = acc[ri + 24] + bs[48 + jj + e];
          float gi, gf, gg, go;
          if (ACC) {
            gi = sigmoid_acc(zi); gf = sigmoid_acc(zf); gg = tanhf(zg); go = sigmoid_acc(zo);
          } else {      // sigmoid(z) = 0.5 tanh(z/2) + 0.5; the 1/2 is folded into the packed weights and bias
            gi = fmaf(0.5f, tanh_approx(zi), 0.5f);
            gf = fmaf(0.5f, tanh_approx(zf), 0.5f);
            gg = tanh_approx(zg);
            go = fmaf(0.5f, tanh_approx(zo), 0.5f);
          }
          cn[e] = fmaf(gf, e ? cprev.y : cprev.x, gi * gg);
          hv[e] = go * (ACC ? tanhf(cn[e]) : tanh_approx(cn[e]));
          gv[0][e] = gi; gv[1][e] = gf; gv[2][e] = gg; gv[3][e] = go;
        }
        *reinterpret_cast<float2*>(cs + jj) = make_float2(cn[0], cn[1]);
        if (valid) {
          const long hoff = ((long)(p.t + 1) * p.Bp + b) * p.H + j;
          const uint32_t w = pack_bf16x2(hv[0], hv[1]);
          st_b32(p.hseq + hoff, w);
          if (p.hseq_lo)        // bf16x3: h = hi + lo with |lo| <= 2^-9 |h|
            st_b32(p.hseq_lo + hoff, pack_bf16x2(hv[0] - bf16_lo(w), hv[1] - bf16_hi(w)));
          if (p.hmseq) {
            float mk[4];
            rec_mask4(p.rkey, p.row0 + b, p.H, j, mk);
            const float m0 = mk[j & 3] * hv[0], m1 = mk[(j & 3) + 1] * hv[1];
            const uint32_t wm = pack_bf16x2(m0, m1);
            st_b32(p.hmseq + hoff, wm);
            if constexpr (ACC) {      // bf16x3: the masked h is the A operand of the lo(h) hi(W) pass
              if (p.hmseq_lo) st_b32(p.hmseq_lo + hoff, pack_bf16x2(m0 - bf16_lo(wm), m1 - bf16_hi(wm)));
            }
          }
          if (p.gates) {
            const long sb = (((long)p.t * p.NRT + rt) * p.NB16 + gblk);
            __nv_bfloat16* gp = p.gates + (((sb * 4 + 0) * 4 + (m >> 5)) * 32 + (m & 31)) * 16 + jj;
            const long gstride = 4L * 32 * 16;           // between gates
#pragma unroll
            for (int g = 0; g < 4; ++g) st_b32(gp + g * gstride, pack_bf16x2(gv[g][0], gv[g][1]));
            st_b32(p.cst + ((sb * 4 + (m >> 5)) * 32 + (m & 31)) * 16 + jj, pack_bf16x2(cn[0], cn[1]));
          }
        }
      }
    }
  }
}

// ---- EPI_GRU_FWD: Keras reset-after GRU (rnn_point_estimate.py:89-98; the SIMT gru_pointwise_fwd_kernel) -----------
// Accumulator columns of a tile: [16-unit block][slot z|r|n_x|n_h][16], slot registers as in epi_fwd.  n_x holds only
// x_t W_h and n_h only h_{t-1} U_h (gpack_kernel zeroes the other half of their K range), so that
//   z = sig(acc_z + b_z), r = sig(acc_r + b_r), n = tanh(acc_nx + b_nx + r (acc_nh + b_nh)), h_t = z h_{t-1} + (1 - z) n
// with h_{t-1} the unmasked state carried in fp32 in cstate.  Forward-only: no gate state is saved.
template <bool ACC>
__device__ __forceinline__ void epi_gru_fwd(const EpiParams& p, const float (&acc)[128], Frag f, int rt, int by,
                                            const float* bias_s) {
  constexpr int U = 64;                             // hidden units of this tile
  // The bias values and Philox quad indices of a thread do not change between the steps of a persistent launch.  Hoisted
  // out of the step loop, they stay live next to the 128 accumulators and spill (about 0.9 KB of spill stores per thread
  // at CUDA 12.9).  The empty asm statements make them opaque to the compiler, so they are re-read and recomputed per step.
  const int unit0 = by * U, mm0 = f.m0;
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    const int m = mm0 + 8 * h;
    const long b = (long)rt * 128 + m;
    const bool valid = b < p.B;
#pragma unroll
    for (int blk = 0; blk < U / 16; ++blk) {
      const int gblk = (unit0 >> 4) + blk;
      float* cs = p.cstate + ((((long)rt * p.NB16 + gblk) * 4 + (m >> 5)) * 32 + (m & 31)) * 16;
      const float* bs = bias_s + blk * 64;
      asm volatile("" : "+l"(bs));
#pragma unroll
      for (int q = 0; q < 2; ++q) {
        const int jj = 8 * q + 2 * f.cq;
        const int j = unit0 + blk * 16 + jj;
        const float2 hprev = p.t > 0 ? *reinterpret_cast<const float2*>(cs + jj) : make_float2(0.f, 0.f);
        float hv[2];
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          const int ri = 32 * blk + 4 * q + 2 * h + e;
          const float az = acc[ri] + bs[jj + e];
          const float ar = acc[ri + 8] + bs[16 + jj + e];
          const float anx = acc[ri + 16] + bs[32 + jj + e];
          const float anh = acc[ri + 24] + bs[48 + jj + e];
          float gz, gr, gn;
          if (ACC) {
            gz = sigmoid_acc(az); gr = sigmoid_acc(ar); gn = tanhf(fmaf(gr, anh, anx));
          } else {      // z and r pre-scaled by 1/2 in the packed weights and bias, as the LSTM's sigmoid gates
            gz = fmaf(0.5f, tanh_approx(az), 0.5f);
            gr = fmaf(0.5f, tanh_approx(ar), 0.5f);
            gn = tanh_approx(fmaf(gr, anh, anx));
          }
          hv[e] = fmaf(gz, (e ? hprev.y : hprev.x) - gn, gn);
        }
        *reinterpret_cast<float2*>(cs + jj) = make_float2(hv[0], hv[1]);
        if (valid) {
          const long hoff = ((long)(p.t + 1) * p.Bp + b) * p.H + j;
          const uint32_t w = pack_bf16x2(hv[0], hv[1]);
          st_b32(p.hseq + hoff, w);
          if (ACC && p.hseq_lo) st_b32(p.hseq_lo + hoff, pack_bf16x2(hv[0] - bf16_lo(w), hv[1] - bf16_hi(w)));
          if (p.hmseq) {
            float mk[4];
            uint64_t quad = (uint64_t)(p.row0 + b) * (uint64_t)(p.H / 4) + (uint64_t)(j / 4);    // rec_mask4
            asm volatile("" : "+l"(quad));
            dropout_quad(p.rkey, quad, mk);
            const float hm0 = mk[j & 3] * hv[0], hm1 = mk[(j & 3) + 1] * hv[1];
            const uint32_t wm = pack_bf16x2(hm0, hm1);
            st_b32(p.hmseq + hoff, wm);
            if (ACC && p.hmseq_lo) st_b32(p.hmseq_lo + hoff, pack_bf16x2(hm0 - bf16_lo(wm), hm1 - bf16_hi(wm)));
          }
        }
      }
    }
  }
}

// ---- EPI_BWD: BPTT pointwise algebra of step t (SURVEY App. A.4) ----------------------------------------------
// Accumulator columns: hidden units unit0 .. unit0+BN-1 in order (rec = dz_{t+1} U^T, before the recurrent mask).
// Every thread handles its fragment's pairs of adjacent units: two per packed bf16x2 word of the saved state.
template <int BN>
__device__ __forceinline__ void epi_bwd(const EpiParams& p, const float (&acc)[BN / 2], Frag f, int rt, int by) {
  const int unit0 = by * BN;
  const long gstride = 4L * 32 * 16;
  const long tstride_c = (long)p.NRT * p.NB16 * 4 * 32 * 16;     // cst elements per time step
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    const int m = f.m0 + 8 * h;
    const long b = (long)rt * 128 + m;
    const bool valid = b < p.B;
    const int q = m >> 5, ln = m & 31;
    __nv_bfloat16* dzr = p.dz + ((long)p.t * p.Bp + b) * 4 * p.H;
#pragma unroll
    for (int J = 0; J < BN / 8; ++J) {
      const int j = unit0 + 8 * J + 2 * f.cq;
      const int gblk = j >> 4, jj = j & 15;
      float* dcs = p.dcstate + ((((long)rt * p.NB16 + gblk) * 4 + q) * 32 + ln) * 16 + jj;
      uint32_t i2 = 0, f2 = 0, g2 = 0, o2 = 0, c2 = 0, cp2 = 0, d2 = 0;
      float2 dcc = make_float2(0.f, 0.f);
      if (valid) {        // rows beyond the batch load nothing and store zero dz
        const long sb = (((long)p.t * p.NRT + rt) * p.NB16 + gblk);
        const __nv_bfloat16* gp = p.gates + (((sb * 4 + 0) * 4 + q) * 32 + ln) * 16 + jj;
        const __nv_bfloat16* cp_ = p.cst + ((sb * 4 + q) * 32 + ln) * 16 + jj;
        i2 = ld_b32(gp);
        f2 = ld_b32(gp + gstride);
        g2 = ld_b32(gp + 2 * gstride);
        o2 = ld_b32(gp + 3 * gstride);
        c2 = ld_b32(cp_);
        cp2 = p.t > 0 ? ld_b32(cp_ - tstride_c) : 0u;
        d2 = ld_b32(p.dhout + ((long)p.t * p.Bp + b) * p.H + j);
        if (p.t < p.T - 1) dcc = *reinterpret_cast<const float2*>(dcs);
      }
      float rec0 = 0.f, rec1 = 0.f;
      if (p.has_rec) {
        rec0 = acc[4 * J + 2 * h];
        rec1 = acc[4 * J + 2 * h + 1];
        if (p.use_rec) {
          float mk[4];
          rec_mask4(p.rkey, p.row0 + b, p.H, j, mk);
          rec0 *= mk[j & 3];
          rec1 *= mk[(j & 3) + 1];
        }
      }
      // Gate-gradient algebra in packed bf16x2 (all operands arrive packed, dz leaves packed); only the carried
      // dLoss/dc stays in fp32.  SURVEY App. A.4.
      const uint32_t dh2 = add_bf16x2(d2, pack_bf16x2(rec0, rec1));
      const uint32_t tc2 = tanh_bf16x2(c2);
      const uint32_t omtc2 = fma_bf16x2(neg_bf16x2(tc2), tc2, BF16X2_ONE);        // 1 - tanh(c)^2
      const uint32_t t1 = mul_bf16x2(mul_bf16x2(dh2, o2), omtc2);                 // dh * o * (1 - tc^2)
      const float dcn0 = dcc.x + bf16_lo(t1);
      const float dcn1 = dcc.y + bf16_hi(t1);
      const uint32_t dcn2 = pack_bf16x2(dcn0, dcn1);
      const uint32_t omi = fma_bf16x2(neg_bf16x2(i2), i2, i2);                    // i (1 - i)
      const uint32_t omf = fma_bf16x2(neg_bf16x2(f2), f2, f2);                    // f (1 - f)
      const uint32_t omg = fma_bf16x2(neg_bf16x2(g2), g2, BF16X2_ONE);            // 1 - g^2
      const uint32_t omo = fma_bf16x2(neg_bf16x2(o2), o2, o2);                    // o (1 - o)
      uint32_t zi = mul_bf16x2(dcn2, mul_bf16x2(g2, omi));
      uint32_t zf = mul_bf16x2(dcn2, mul_bf16x2(cp2, omf));
      uint32_t zg = mul_bf16x2(dcn2, mul_bf16x2(i2, omg));
      uint32_t zo = mul_bf16x2(mul_bf16x2(dh2, tc2), omo);
      if (valid) {
        *reinterpret_cast<float2*>(dcs) = make_float2(dcn0 * bf16_lo(f2), dcn1 * bf16_hi(f2));
      } else {          // rows beyond the batch: dz exactly zero (the weight-gradient GEMM sums over all rows)
        zi = zf = zg = zo = 0u;
      }
      st_b32(dzr + j, zi);
      st_b32(dzr + p.H + j, zf);
      st_b32(dzr + 2L * p.H + j, zg);
      st_b32(dzr + 3L * p.H + j, zo);
    }
  }
}

// ---- EPI_STORE: accumulator -> bf16 row-major ---------------------------------------------------------------------
template <int BN>
__device__ __forceinline__ void epi_store(const EpiParams& p, const float (&acc)[BN / 2], Frag f, long row0, int by) {
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    __nv_bfloat16* o = p.out + (row0 + f.m0 + 8 * h) * p.ldc + (long)by * BN + 2 * f.cq;
#pragma unroll
    for (int J = 0; J < BN / 8; ++J) st_b32(o + 8 * J, pack_bf16x2(acc[4 * J + 2 * h], acc[4 * J + 2 * h + 1]));
  }
}

// ---- EPI_HEAD: Dense + weighted MSE + dLoss/dpred on the accumulator of pred = y Wo (N = 16) ---------------------------
// One CTA = one 128-row tile (t, rt) of the time-major head input; the accumulator is staged in shared memory so that
// threads 0..127 own one row each.  (rnn_point_estimate.py:105; model_utils/losses.py:55-135; SURVEY App. A.3)
constexpr int GH_O = 16;
constexpr int GH_PART = GH_O + 4;      // dbo | s0 s1 s2
__device__ __forceinline__ void epi_head(const EpiParams& p, const float (&acc)[8], Frag f, float* rows_s, float* red_s) {
  const int tid = threadIdx.x;
#pragma unroll
  for (int i = 0; i < 8; ++i) rows_s[(f.m0 + 8 * ((i >> 1) & 1)) * 17 + 8 * (i >> 2) + 2 * f.cq + (i & 1)] = acc[i];
  if (tid < GH_PART) red_s[tid] = 0.f;
  named_bar_sync(1, 256);
  if (tid >= 128) return;
  const int tile = blockIdx.x;
  const int t = tile / p.NRT, rt = tile % p.NRT;
  const int m = tid;
  const long b = (long)rt * 128 + m;
  const bool valid = b < p.B;
  const long r = b * p.T + t;          // row of the caller's [B][T][O] tensors
  float yt[GH_O];
#pragma unroll
  for (int k = 0; k < GH_O; ++k) yt[k] = 0.f;
  if (p.hy && valid)
    for (int k = 0; k < p.hO; ++k) yt[k] = p.hy[r * p.hO + k];
  float pr[GH_O];
#pragma unroll
  for (int k = 0; k < GH_O; ++k) pr[k] = (k < p.hO) ? rows_s[m * 17 + k] + __ldg(p.hbo + k) : 0.f;
  if (p.hpreds && valid)
    for (int k = 0; k < p.hO; ++k) p.hpreds[r * p.hO + k] = pr[k];
  if (!p.hy) return;
  LossWeights lw = {0.f, 0.f, 0.f};
  if (p.htrain) lw = loss_weights(p.hp1, p.hp2, p.hO, p.hdenom[1], p.hdenom[0], p.hrw);
  const float mk = (row_mask(yt, GH_O) && valid) ? 1.f : 0.f;
  const float wb = valid ? row_weight(p.hrw, b) : 0.f;
  float s0 = 0.f, s1 = 0.f, s2 = 0.f;
  float dp[GH_O] = {};
  point_loss_row<GH_O>(pr, yt, p.hO, valid, mk, wb, t == p.T - 1, p.htarget, lw, p.htrain, dp, s0, s1, s2);
  if (p.htrain) {       // every row of the tile is written (zeros beyond the batch): the dy / dWo GEMMs run over all rows
    uint32_t w[8];
#pragma unroll
    for (int e = 0; e < 8; ++e) w[e] = pack_bf16x2(dp[2 * e], dp[2 * e + 1]);
    st_global_v8(p.hdpb + ((long)t * p.Bp + b) * 64, w);
  }
  flush_loss_sums(red_s, GH_O, 0, s0, s1, s2, dp, p.htrain);
  named_bar_sync(2, 128);
  if (m < GH_PART) p.hpartial[(long)m * gridDim.x + blockIdx.x] = red_s[m];
}

// ---- EPI_HEAD_UQ: the two heads of RNNUqRangeEstimate on the accumulator of y [Wo | Wv] (N = 32), forward only -------
// pred = y Wo + bo, var = max(softplus(y Wv + bv), 1e-6) (rnn_uq_range_estimate.py:104-108, custom_layers.py:12-13).
// Staged in shared memory like epi_head so that threads 0..127 own one row each and write its O outputs contiguously.
__device__ __forceinline__ void epi_head_uq(const EpiParams& p, const float (&acc)[16], Frag f, float* rows_s) {
  constexpr int LD = 2 * GH_O + 1;
#pragma unroll
  for (int i = 0; i < 16; ++i) rows_s[(f.m0 + 8 * ((i >> 1) & 1)) * LD + 8 * (i >> 2) + 2 * f.cq + (i & 1)] = acc[i];
  named_bar_sync(1, 256);
  const int m = threadIdx.x;
  if (m >= 128) return;
  const int t = (int)blockIdx.x / p.NRT, rt = (int)blockIdx.x % p.NRT;
  const long b = (long)rt * 128 + m;
  if (b >= p.B) return;
  const long r = b * p.T + t;          // row of the caller's [B][T][O] tensors
  for (int k = 0; k < p.hO; ++k) {
    p.hpreds[r * p.hO + k] = rows_s[m * LD + k] + __ldg(p.hbo + k);
    p.hvar[r * p.hO + k] = fmaxf(softplus_f(rows_s[m * LD + GH_O + k] + __ldg(p.hbv + k)), 1e-6f);
  }
}

template <int BN, int EPI>
__global__ void __launch_bounds__(GSmem<BN, EPI>::THREADS, GSmem<BN, EPI>::CTAS_PER_SM)
    tile_gemm_kernel(GArgs g, EpiParams ep, const __grid_constant__ CUtensorMap tmA0,
                     const __grid_constant__ CUtensorMap tmA1, const __grid_constant__ CUtensorMap tmA2,
                     const __grid_constant__ CUtensorMap tmA3, const __grid_constant__ CUtensorMap tmB0,
                     const __grid_constant__ CUtensorMap tmB1) {
  using S = GSmem<BN, EPI>;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint64_t* full = reinterpret_cast<uint64_t*>(smem + S::BARS);
  uint64_t* empty = full + S::NS;
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  __shared__ float red_s[EPI == EPI_HEAD ? GH_PART : 1];
  __shared__ float bias_s[epi_is_fwd(EPI) ? BN : 1];
  if constexpr (epi_is_fwd(EPI))
    for (int i = tid; i < BN; i += S::THREADS) bias_s[i] = ep.bias[blockIdx.y * BN + i];    // weights: not the predecessor's

  int total_kb = 0;
  for (int i = 0; i < g.n_seg; ++i) total_kb += g.seg[i].n_kb;

  if (tid == 0) {
    for (int s = 0; s < S::NS; ++s) {
      mbar_init(&full[s], 1);
      mbar_init(&empty[s], 8);               // one arrive per consumer warp
    }
    fence_mbar_init();
  }
  __syncthreads();
  const int bx = g.lin_cols > 0 ? (int)blockIdx.x / g.lin_cols : (int)blockIdx.x;      // row-tile / column-tile coordinates
  const int by = g.lin_cols > 0 ? (int)blockIdx.x % g.lin_cols : (int)blockIdx.y;

  // Programmatic dependent launch (the recurrence steps are launched with the stream-serialization attribute): this
  // kernel's CTAs are dispatched while the previous step's grid drains.  Everything above (barriers) and the B
  // operand (weights: packed long before the previous step) of the first ring stages is independent of it; the A
  // operand and every state the epilogue reads were written by the previous step, so all threads wait here first.
  // launch_dependents comes AFTER the wait: when the next grid starts, this one has seen its predecessor complete, so
  // by induction only the immediate predecessor can still be running.
  const int n_steps = g.n_steps > 1 ? g.n_steps : 1;
  const unsigned int n_cta = gridDim.y;             // CTAs of this row-tile group
  if (warp == 8) {
    if (lane == 0) {
      const int brow = g.b_row_base + BN * by;
      for (int it = 0; it < n_steps; ++it) {
        const int arow = g.a_row_base + it * g.row_step + 128 * (bx + g.rt_off);
        const int gi0 = it * total_kb;               // ring position of this step's first k-block
        {   // B operand (weights) of the first NS stages of the step, before the dependency wait
          int i = 0;
          for (int sg = 0; sg < g.n_seg && i < S::NS; ++sg) {
            const GSeg sgm = g.seg[sg];
            const CUtensorMap* mb = sgm.b_map == 0 ? &tmB0 : &tmB1;
            for (int kb = 0; kb < sgm.n_kb && i < S::NS; ++kb, ++i) {
              const int gi = gi0 + i, st_ = gi % S::NS;
              if (gi >= S::NS) mbar_wait(&empty[st_], ((gi / S::NS) - 1) & 1);
              mbar_arrive_expect_tx(&full[st_], S::STAGE);
              tma_load_2d(smem + st_ * S::STAGE + S::A_BYTES, mb, &full[st_], sgm.b_col0 + kb * 64, brow);
            }
          }
        }
        if (it == 0) {
          pdl_sync();
        } else {
          // every CTA of the row-tile group has published step it-1 (generic-proxy stores, fenced before the count went up)
          const long long spin0 = clock64();
          while (ld_acquire_gpu(g.gbar + blockIdx.x) < (unsigned int)it * n_cta) {
            // the host only takes this mode when all CTAs fit on the machine at once; should a peer never arrive
            // (SMs held by somebody else), fail the launch after ~2 s instead of hanging the device
            if (clock64() - spin0 > 4000000000LL) __trap();
          }
          fence_proxy_async_global();
        }
        int i = 0;
        for (int sg = 0; sg < g.n_seg; ++sg) {
          const GSeg sgm = g.seg[sg];
          const CUtensorMap* ma = sgm.a_map == 0 ? &tmA0 : (sgm.a_map == 1 ? &tmA1 : (sgm.a_map == 2 ? &tmA2 : &tmA3));
          const CUtensorMap* mb = sgm.b_map == 0 ? &tmB0 : &tmB1;
          for (int kb = 0; kb < sgm.n_kb; ++kb, ++i) {
            const int gi = gi0 + i, s = gi % S::NS;
            uint8_t* st = smem + s * S::STAGE;
            if (i >= S::NS) {
              mbar_wait(&empty[s], ((gi / S::NS) - 1) & 1);
              mbar_arrive_expect_tx(&full[s], S::STAGE);
              tma_load_2d(st + S::A_BYTES, mb, &full[s], sgm.b_col0 + kb * 64, brow);
            }
            tma_load_2d(st, ma, &full[s], sgm.a_col0 + kb * 64, arow);
          }
        }
      }
    } else {
      pdl_sync();
    }
  } else if (warp < 8) {
    pdl_sync();
    const int wg = warp >> 2;
    const Frag f{64 * wg + 16 * (warp & 3) + (lane >> 2), lane & 3};
    const int rt = bx + g.rt_off;                    // 128-row tile index
    const int t_first = ep.t;
    float acc[BN / 2];
    for (int it = 0; it < n_steps; ++it) {
      ep.t = t_first + it * g.t_step;
      for (int i = 0; i < total_kb; ++i) {
        const int gi = it * total_kb + i, s = gi % S::NS;
        mbar_wait(&full[s], (gi / S::NS) & 1);
        uint8_t* st = smem + s * S::STAGE;
        wgmma_fence();
#pragma unroll
        for (int k16 = 0; k16 < 4; ++k16) {
          const uint64_t db = make_smem_desc(smem_u32(st + S::A_BYTES) + k16 * 32, 0, 1024, LAYOUT_SW128);
          const uint64_t da = make_smem_desc(smem_u32(st + wg * 8192) + k16 * 32, 0, 1024, LAYOUT_SW128);
          wgmma_bn<BN>(acc, da, db, (i | k16) != 0);
        }
        wgmma_commit();
        wgmma_wait<1>();                             // the previous stage's MMAs are complete: release it
        if (i > 0 && lane == 0) mbar_arrive(&empty[(gi - 1) % S::NS]);
      }
      wgmma_wait<0>();
      fence_regs(acc);
      if (total_kb > 0 && lane == 0) mbar_arrive(&empty[(it * total_kb + total_kb - 1) % S::NS]);
      if constexpr (EPI == EPI_HEAD) {
        epi_head(ep, acc, f, reinterpret_cast<float*>(smem + S::HEAD_ROWS), red_s);
      } else if constexpr (EPI == EPI_HEAD_UQ) {
        epi_head_uq(ep, acc, f, reinterpret_cast<float*>(smem + S::HEAD_ROWS));
      } else if ((long)rt * 128 < ep.Bp || EPI == EPI_STORE) {
        if constexpr (EPI == EPI_FWD) epi_fwd<false>(ep, acc, f, rt, by, bias_s);
        if constexpr (EPI == EPI_FWD_ACC) epi_fwd<true>(ep, acc, f, rt, by, bias_s);
        if constexpr (EPI == EPI_GRU_FWD) epi_gru_fwd<false>(ep, acc, f, rt, by, bias_s);
        if constexpr (EPI == EPI_GRU_FWD_ACC) epi_gru_fwd<true>(ep, acc, f, rt, by, bias_s);
        if constexpr (EPI == EPI_BWD) epi_bwd<BN>(ep, acc, f, rt, by);
        if constexpr (EPI == EPI_STORE) epi_store<BN>(ep, acc, f, (long)g.a_row_base + 128L * rt, by);
      }
      if (n_steps > 1) {
        // end of a step: both consumer warpgroups are done with the accumulator and have issued their stores; one
        // thread makes them visible device-wide and counts the CTA in (the pattern of a cooperative grid sync)
        named_bar_sync(2, 256);
        if (tid == 0) {
          __threadfence();
          atomicAdd(g.gbar + blockIdx.x, 1u);
        }
      }
    }
  }
}

// =============================================================================================
// Weight gradients D = A^T B over the T*Bp time-major rows: wgrad_gemm (tc_shared.h) and the reductions of its partials
// =============================================================================================
// dst[row][n] = sum_z partial[z][row][n] for row < Mvalid (dst row-major [Mvalid][Ntot])
// (rows row_first .. row_first + Mvalid - 1 of the partials)
__global__ void gwgrad_reduce_kernel(int S, int Mvalid, int Mpad, int Ntot, const float* __restrict__ partial,
                                     float* __restrict__ dst, int row_first) {
  const long idx = ((long)blockIdx.x * blockDim.x + threadIdx.x) * 4;
  if (idx >= (long)Mvalid * Ntot) return;
  float4 s = make_float4(0.f, 0.f, 0.f, 0.f);
  for (int z = 0; z < S; ++z) {
    const float4 v = *reinterpret_cast<const float4*>(partial + (long)z * Mpad * Ntot + (long)row_first * Ntot + idx);
    s.x += v.x; s.y += v.y; s.z += v.z; s.w += v.w;
  }
  *reinterpret_cast<float4*>(dst + idx) = s;
}

// =============================================================================================
// Small streaming kernels
// =============================================================================================
// x f32 [B][T][F] -> in0 bf16 [T][Bp][Ipad] (+ low halves for bf16x3); 8 columns per thread, padding columns zero.
// `ones`: column F (the first padding column) is set to 1 -- the weights of the padding rows are zero, so the forward GEMM
// does not see it, and the weight-gradient GEMM in0^T dz then delivers db = colsum(dz) of the first layer as its row F.
__global__ void gcast_x_kernel(int B, int T, int F, int Bp, int Ipad, const float* __restrict__ x,
                               __nv_bfloat16* __restrict__ o, __nv_bfloat16* __restrict__ o_lo, int ones) {
  const int c8 = Ipad / 8;
  const long idx = (long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= (long)B * T * c8) return;
  const int c = (int)(idx % c8);
  const long r = idx / c8;
  const int t = (int)(r % T);
  const long b = r / T;
  float v[8];
#pragma unroll
  for (int e = 0; e < 8; ++e) {
    const int f = c * 8 + e;
    v[e] = (f < F) ? x[(b * T + t) * F + f] : ((ones && f == F) ? 1.f : 0.f);
  }
  uint4 w;
  w.x = pack_bf16x2(v[0], v[1]); w.y = pack_bf16x2(v[2], v[3]); w.z = pack_bf16x2(v[4], v[5]); w.w = pack_bf16x2(v[6], v[7]);
  const long off = ((long)t * Bp + b) * Ipad + c * 8;
  *reinterpret_cast<uint4*>(o + off) = w;
  if (o_lo) {
    uint4 l;
    l.x = pack_bf16x2(v[0] - bf16_lo(w.x), v[1] - bf16_hi(w.x));
    l.y = pack_bf16x2(v[2] - bf16_lo(w.y), v[3] - bf16_hi(w.y));
    l.z = pack_bf16x2(v[4] - bf16_lo(w.z), v[5] - bf16_hi(w.z));
    l.w = pack_bf16x2(v[6] - bf16_lo(w.w), v[7] - bf16_hi(w.w));
    *reinterpret_cast<uint4*>(o_lo + off) = l;
  }
}

// Packed operands of one layer.
//   Wf  [4H][Kp]  forward B operand, K = [h (H) | input (Ipad)], row n = tile*256 + blk*64 + gate*16 + jj  <->  gate column
//                 gate*H + tile*64 + blk*16 + jj of [U; W]; sigmoid gates (i, f, o) pre-scaled by `hs` (0.5, or 1 when accurate)
//   Ub  [H][4H]   backward B operand = recurrent_kernel as it is (rec = dz U^T)
//   Wb  [I][4H]   dLoss/d(input) B operand = kernel as it is (layers above the first)
//   biasp [4H]    bias in Wf's row order, same pre-scale
// GRU (forward only): the four gate slots of a 16-unit block are z | r | n_x | n_h (Keras blocks z | r | h of W, U [I|H][3H]
// and bias [2][3H]).  n_x takes only W_h (zero rows for K < H) and n_h only U_h (zero rows for K >= H), so that the reset
// gate can scale h_{t-1} U_h + b_rh alone; z and r take the pre-scale `hs`, their bias is the sum of both bias rows,
// n_x takes b[0]_h and n_h b[1]_h.  The zero blocks cost (H + I) H of the (H + Ipad) 4H MACs; the GEMM keeps the LSTM's
// shape.
struct GPackArgs {
  int H, I, Ipad, Kp, gru;
  float hs, eps;
  const float *W, *U, *bias, *gamma, *beta, *mean, *var;
  __nv_bfloat16 *Wf, *Wf_lo, *Ub, *Wb;
  float* biasp;
  float* bn;          // [4][H]: a = gamma * inv | b = beta - mean * a | mean | inv   (BN as the affine map it is here)
};
__global__ void gpack_kernel(GPackArgs a) {
  const long idx = (long)blockIdx.x * blockDim.x + threadIdx.x;
  const int H = a.H;
  const long nWf = (long)4 * H * a.Kp;
  if (idx < nWf) {
    const int k = (int)(idx % a.Kp);
    const int n = (int)(idx / a.Kp);
    const int tile = n / 256, blk = (n % 256) / 64, gate = (n % 64) / 16, jj = n % 16;
    const int u = tile * 64 + blk * 16 + jj;
    float v = 0.f;
    if (a.gru) {
      const int col = (gate < 2 ? gate : 2) * H + u;
      const float sc = (gate < 2) ? a.hs : 1.0f;
      if (k < H) {
        if (gate != 2) v = sc * a.U[(long)k * 3 * H + col];
      } else if (k - H < a.I) {
        if (gate != 3) v = sc * a.W[(long)(k - H) * 3 * H + col];
      }
    } else {
      const int col = gate * H + u;
      const float sc = (gate == 2) ? 1.0f : a.hs;
      if (k < H) v = sc * a.U[(long)k * 4 * H + col];
      else if (k - H < a.I) v = sc * a.W[(long)(k - H) * 4 * H + col];
    }
    const __nv_bfloat16 hi = __float2bfloat16(v);
    a.Wf[idx] = hi;
    if (a.Wf_lo) a.Wf_lo[idx] = __float2bfloat16(v - __bfloat162float(hi));
  }
  if (idx < (long)H * 4 * H && a.Ub) a.Ub[idx] = __float2bfloat16(a.U[idx]);
  if (idx < (long)a.I * 4 * H && a.Wb) a.Wb[idx] = __float2bfloat16(a.W[idx]);
  if (idx < 4 * H) {
    const int n = (int)idx;
    const int tile = n / 256, blk = (n % 256) / 64, gate = (n % 64) / 16, jj = n % 16;
    const int u = tile * 64 + blk * 16 + jj;
    if (a.gru)
      a.biasp[n] = gate < 2 ? a.hs * (a.bias[gate * H + u] + a.bias[3 * H + gate * H + u])
                            : a.bias[(gate == 2 ? 0 : 3 * H) + 2 * H + u];
    else
      a.biasp[n] = ((gate == 2) ? 1.0f : a.hs) * a.bias[gate * H + u];
  }
  if (idx < H) {
    const int j = (int)idx;
    const float inv = 1.0f / sqrtf(a.var[j] + a.eps);
    const float ga = a.gamma[j] * inv;
    a.bn[j] = ga;
    a.bn[H + j] = a.beta[j] - a.mean[j] * ga;
    a.bn[2 * H + j] = a.mean[j];
    a.bn[3 * H + j] = inv;
  }
}

// Head operands: WoT [16][H] (B operand of pred = y Wo: row = output k, K = hidden) and WoS [H][64] (B operand of
// dy = dpred Wo^T: row = hidden unit, K = output k, zero beyond O; null: not packed).  uq handles pack the variance
// head's Wv into rows 16..31 of WoT with a second call.
__global__ void gpack_head_kernel(int H, int O, const float* __restrict__ Wo, __nv_bfloat16* __restrict__ WoT,
                                  __nv_bfloat16* __restrict__ WoS) {
  const int idx = blockIdx.x * blockDim.x + threadIdx.x;
  if (idx < 16 * H) {
    const int k = idx / H, j = idx % H;
    WoT[idx] = __float2bfloat16(k < O ? Wo[j * O + k] : 0.f);
  }
  if (WoS && idx < H * 64) {
    const int j = idx / 64, k = idx % 64;
    WoS[idx] = __float2bfloat16(k < O ? Wo[j * O + k] : 0.f);
  }
}

// dWo[j][k] = sum_z partial[z][j][k] (k < O) from the weight-gradient GEMM of the head (N padded to 256)
__global__ void ghead_wo_reduce_kernel(int S, int H, int O, int Mpad, const float* __restrict__ partial,
                                       float* __restrict__ gWo) {
  const int idx = blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= H * O) return;
  const int j = idx / O, k = idx % O;
  float s = 0.f;
  for (int z = 0; z < S; ++z) s += partial[((long)z * Mpad + j) * 256 + k];
  gWo[idx] = s;
}

// y = Dropout(BN(h)) (rnn_point_estimate.py:88-89; BN is the inference affine in both modes, SURVEY App. B #1):
// hseq slots 1..T -> in_next [T][Bp][H] (+ low halves for bf16x3).  8 columns per thread.
__global__ void __launch_bounds__(256)
    gbn_drop_fwd_kernel(int B, int T, int H, int Bp, const __nv_bfloat16* __restrict__ hseq,
                        const __nv_bfloat16* __restrict__ hseq_lo, const float* __restrict__ bn, int use_dropout,
                        DropoutKey key, int64_t row0, __nv_bfloat16* __restrict__ y, __nv_bfloat16* __restrict__ y_lo) {
  const int c8 = H / 8;
  const long idx = (long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= (long)T * B * c8) return;
  const int c = (int)(idx % c8);
  const long r = idx / c8;
  const long b = r % B;
  const int t = (int)(r / B);
  const long off = ((long)t * Bp + b) * H + c * 8;
  const uint4 hw = *reinterpret_cast<const uint4*>(hseq + off + (long)Bp * H);      // slot t+1
  float hv[8] = {bf16_lo(hw.x), bf16_hi(hw.x), bf16_lo(hw.y), bf16_hi(hw.y), bf16_lo(hw.z), bf16_hi(hw.z), bf16_lo(hw.w), bf16_hi(hw.w)};
  if (hseq_lo) {
    const uint4 lw = *reinterpret_cast<const uint4*>(hseq_lo + off + (long)Bp * H);
    const float lv[8] = {bf16_lo(lw.x), bf16_hi(lw.x), bf16_lo(lw.y), bf16_hi(lw.y), bf16_lo(lw.z), bf16_hi(lw.z), bf16_lo(lw.w), bf16_hi(lw.w)};
#pragma unroll
    for (int e = 0; e < 8; ++e) hv[e] += lv[e];
  }
  float mk[8];
  dropout8(key, use_dropout, row0 + b, t, T, H, c, mk);
  const float4 a0 = __ldg(reinterpret_cast<const float4*>(bn + c * 8)), a1 = __ldg(reinterpret_cast<const float4*>(bn + c * 8 + 4));
  const float4 b0 = __ldg(reinterpret_cast<const float4*>(bn + H + c * 8)), b1 = __ldg(reinterpret_cast<const float4*>(bn + H + c * 8 + 4));
  const float av[8] = {a0.x, a0.y, a0.z, a0.w, a1.x, a1.y, a1.z, a1.w};
  const float bv[8] = {b0.x, b0.y, b0.z, b0.w, b1.x, b1.y, b1.z, b1.w};
  float o[8];
#pragma unroll
  for (int e = 0; e < 8; ++e) o[e] = fmaf(av[e], hv[e], bv[e]) * mk[e];
  uint4 w;
  w.x = pack_bf16x2(o[0], o[1]); w.y = pack_bf16x2(o[2], o[3]); w.z = pack_bf16x2(o[4], o[5]); w.w = pack_bf16x2(o[6], o[7]);
  *reinterpret_cast<uint4*>(y + off) = w;
  if (y_lo) {
    uint4 l;
    l.x = pack_bf16x2(o[0] - bf16_lo(w.x), o[1] - bf16_hi(w.x));
    l.y = pack_bf16x2(o[2] - bf16_lo(w.y), o[3] - bf16_hi(w.y));
    l.z = pack_bf16x2(o[4] - bf16_lo(w.z), o[5] - bf16_hi(w.z));
    l.w = pack_bf16x2(o[6] - bf16_lo(w.w), o[7] - bf16_hi(w.w));
    *reinterpret_cast<uint4*>(y_lo + off) = l;
  }
}

// Dropout / BN backward: dhout = dy * mask * gamma * inv; per-CTA partial sums of dgamma, dbeta (SURVEY App. A.4).
// Thread = 8 columns; a CTA of 256 threads holds 256 / (H/8) rows at a time and walks its row range.
constexpr int GBN_ROWS = 64;
__global__ void __launch_bounds__(256)
    gbn_drop_bwd_kernel(int B, int T, int H, int Bp, const __nv_bfloat16* __restrict__ dy,
                        const __nv_bfloat16* __restrict__ hseq, const float* __restrict__ bn, int use_dropout,
                        DropoutKey key, int64_t row0, __nv_bfloat16* __restrict__ dhout, float* __restrict__ partial) {
  extern __shared__ float red[];      // [RL][2H]
  const int c8 = H / 8;
  const int RL = blockDim.x / c8;
  const int c = threadIdx.x % c8, rl = threadIdx.x / c8;
  float g[8], mu[8], inv[8], sg[8], sb[8];
#pragma unroll
  for (int e = 0; e < 8; ++e) {
    const int j = c * 8 + e;
    g[e] = bn[j];
    mu[e] = bn[2 * H + j];
    inv[e] = bn[3 * H + j];
    sg[e] = 0.f;
    sb[e] = 0.f;
  }
  const long rows = (long)T * B;
  const long r0 = (long)blockIdx.x * GBN_ROWS;
  const long r1 = min(rows, r0 + GBN_ROWS);
  if (rl < RL) {
#pragma unroll 2
    for (long r = r0 + rl; r < r1; r += RL) {
      const long b = r % B;
      const int t = (int)(r / B);
      const long off = ((long)t * Bp + b) * H + c * 8;
      const uint4 dw = *reinterpret_cast<const uint4*>(dy + off);
      const uint4 hw = *reinterpret_cast<const uint4*>(hseq + off + (long)Bp * H);
      float d[8] = {bf16_lo(dw.x), bf16_hi(dw.x), bf16_lo(dw.y), bf16_hi(dw.y), bf16_lo(dw.z), bf16_hi(dw.z), bf16_lo(dw.w), bf16_hi(dw.w)};
      const float hv[8] = {bf16_lo(hw.x), bf16_hi(hw.x), bf16_lo(hw.y), bf16_hi(hw.y), bf16_lo(hw.z), bf16_hi(hw.z), bf16_lo(hw.w), bf16_hi(hw.w)};
      if (use_dropout) {
        float mk[8];
        dropout8(key, true, row0 + b, t, T, H, c, mk);
#pragma unroll
        for (int e = 0; e < 8; ++e) d[e] *= mk[e];
      }
      float o[8];
#pragma unroll
      for (int e = 0; e < 8; ++e) {
        sg[e] += d[e] * (hv[e] - mu[e]) * inv[e];
        sb[e] += d[e];
        o[e] = d[e] * g[e];
      }
      uint4 w;
      w.x = pack_bf16x2(o[0], o[1]); w.y = pack_bf16x2(o[2], o[3]); w.z = pack_bf16x2(o[4], o[5]); w.w = pack_bf16x2(o[6], o[7]);
      *reinterpret_cast<uint4*>(dhout + off) = w;
    }
#pragma unroll
    for (int e = 0; e < 8; ++e) {
      red[(long)rl * 2 * H + c * 8 + e] = sg[e];
      red[(long)rl * 2 * H + H + c * 8 + e] = sb[e];
    }
  }
  __syncthreads();
  for (int k = threadIdx.x; k < 2 * H; k += blockDim.x) {
    float sum = 0.f;
    for (int r = 0; r < RL; ++r) sum += red[(long)r * 2 * H + k];
    partial[(long)k * gridDim.x + blockIdx.x] = sum;        // [value][cta]
  }
}

// out[k] = sum over CTAs of partial[k][cta] (one warp per value, fixed order -> deterministic); values [0,n0) go to
// dst0, [n0, n0+n1) to dst1
__global__ void gpartial_reduce_kernel(int n_cta, int n0, int n1, const float* __restrict__ partial,
                                       float* __restrict__ dst0, float* __restrict__ dst1) {
  const int k = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (k >= n0 + n1) return;
  const double s = sum_partials(partial + (long)k * n_cta, 1, n_cta);
  if (lane == 0) {
    if (k < n0) dst0[k] = (float)s;
    else dst1[k - n0] = (float)s;
  }
}

// db = column sums of dz (bf16 [rows][N]) -> partial[column][chunk]; thread = 8 columns (128-bit loads), 4 rows in flight
__global__ void __launch_bounds__(128) gcolsum_kernel(long rows, int N, long rows_per_chunk,
                                                     const __nv_bfloat16* __restrict__ A, float* __restrict__ partial) {
  const int c8 = blockIdx.x * 128 + threadIdx.x;       // group of 8 columns
  if (c8 * 8 >= N) return;
  const long r0 = (long)blockIdx.y * rows_per_chunk, r1 = min(rows, r0 + rows_per_chunk);
  float s[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
  long r = r0;
  for (; r + 4 <= r1; r += 4) {
    uint4 w[4];
#pragma unroll
    for (int u = 0; u < 4; ++u) w[u] = *reinterpret_cast<const uint4*>(A + (r + u) * N + c8 * 8);
#pragma unroll
    for (int u = 0; u < 4; ++u) {
      s[0] += bf16_lo(w[u].x); s[1] += bf16_hi(w[u].x); s[2] += bf16_lo(w[u].y); s[3] += bf16_hi(w[u].y);
      s[4] += bf16_lo(w[u].z); s[5] += bf16_hi(w[u].z); s[6] += bf16_lo(w[u].w); s[7] += bf16_hi(w[u].w);
    }
  }
  for (; r < r1; ++r) {
    const uint4 w = *reinterpret_cast<const uint4*>(A + r * N + c8 * 8);
    s[0] += bf16_lo(w.x); s[1] += bf16_hi(w.x); s[2] += bf16_lo(w.y); s[3] += bf16_hi(w.y);
    s[4] += bf16_lo(w.z); s[5] += bf16_hi(w.z); s[6] += bf16_lo(w.w); s[7] += bf16_hi(w.w);
  }
#pragma unroll
  for (int e = 0; e < 8; ++e) partial[(long)(c8 * 8 + e) * gridDim.y + blockIdx.y] = s[e];
}

// =============================================================================================
// bf16x3 head on y = in[L] (bf16 [T][Bp][H] + low halves, BN / Dropout already applied): pred = y Wo + bo accumulated in
// fp32.  bf16x3 handles are forward-only (gen_supported), so this head only predicts.  One thread per row of a 128-row
// tile (TMA-staged, SW128), Wo broadcast from shared memory.  (rnn_point_estimate.py:105)  uq handles run it a second
// time on the variance head (Wv, bv, softplus_floor = 1: var = max(softplus(y Wv + bv), 1e-6)).
// =============================================================================================
struct GHeadParams {
  int B, T, O, H, Bp, NRT;
  const float *Wo, *bo;
  float* preds;              // [B][T][O] fp32
  const __nv_bfloat16* yin_lo;   // low halves of the head input (row-major, same layout)
  int softplus_floor;
};
__global__ void __launch_bounds__(128, 1) ghead_rows_kernel(GHeadParams p, const __grid_constant__ CUtensorMap tm_y) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* tile = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  const int nkb = p.H / 64;
  float* Wo_s = reinterpret_cast<float*>(tile + (size_t)nkb * 16384);          // [H][16]
  uint64_t* bar = reinterpret_cast<uint64_t*>(Wo_s + (size_t)p.H * GH_O);
  const int tid = threadIdx.x;
  for (int i = tid; i < p.H * GH_O; i += 128) {
    const int j = i / GH_O, k = i % GH_O;
    Wo_s[i] = (k < p.O) ? p.Wo[j * p.O + k] : 0.f;
  }
  if (tid == 0) {
    mbar_init(bar, 1);
    fence_mbar_init();
  }
  __syncthreads();
  const int sw = tid & 7;
  uint32_t phase = 0;
  const int n_tiles = p.T * p.NRT;
  for (int ti = blockIdx.x; ti < n_tiles; ti += gridDim.x) {
    const int t = ti / p.NRT, rt = ti % p.NRT;
    const long b = (long)rt * 128 + tid;
    const bool valid = b < p.B;
    if (tid == 0) {
      mbar_arrive_expect_tx(bar, (uint32_t)nkb * 16384u);
      for (int kb = 0; kb < nkb; ++kb) tma_load_2d(tile + kb * 16384, &tm_y, bar, kb * 64, t * p.Bp + rt * 128);
    }
    const long r = b * p.T + t;          // row of the caller's [B][T][O] tensors
    mbar_wait(bar, phase);
    phase ^= 1;
    const uint8_t* hrow = tile + tid * 128;
    const __nv_bfloat16* lorow = p.yin_lo ? p.yin_lo + ((long)t * p.Bp + b) * p.H : nullptr;
    float pr[GH_O];
#pragma unroll
    for (int k = 0; k < GH_O; ++k) pr[k] = (k < p.O) ? p.bo[k] : 0.f;
#pragma unroll 2
    for (int c = 0; c < p.H / 8; ++c) {
      const uint4 raw = *reinterpret_cast<const uint4*>(hrow + (c >> 3) * 16384 + (((c & 7) ^ sw) << 4));
      const uint32_t hw[4] = {raw.x, raw.y, raw.z, raw.w};
      uint32_t lw[4] = {0u, 0u, 0u, 0u};
      if (lorow && valid) {
        const uint4 l = *reinterpret_cast<const uint4*>(lorow + c * 8);
        lw[0] = l.x; lw[1] = l.y; lw[2] = l.z; lw[3] = l.w;
      }
#pragma unroll
      for (int e = 0; e < 8; ++e) {
        const int j = c * 8 + e;
        const float yv = ((e & 1) ? bf16_hi(hw[e >> 1]) : bf16_lo(hw[e >> 1])) +
                         ((e & 1) ? bf16_hi(lw[e >> 1]) : bf16_lo(lw[e >> 1]));
        const float4* w4 = reinterpret_cast<const float4*>(Wo_s + j * GH_O);
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
    if (p.preds && valid)
      for (int k = 0; k < p.O; ++k) p.preds[r * p.O + k] = p.softplus_floor ? fmaxf(softplus_f(pr[k]), 1e-6f) : pr[k];
    __syncthreads();        // everyone is done with the tile before it is overwritten
  }
}

// Sums the tensor-core head's per-tile partials: loss terms -> {loss, mse_0}, dbo.
__global__ void ghead_reduce_kernel(int n_cta, const float* __restrict__ partial, int O, const float* denom,
                                    const float* rw, float p1, float p2, int train, float* __restrict__ gbo,
                                    float* __restrict__ out2) {
  const int q = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;     // one warp per output value
  const int lane = threadIdx.x & 31;
  if (q >= GH_PART) return;
  const double s = sum_partials(partial + (long)q * n_cta, 1, n_cta);
  if (q < GH_O) {
    if (train && lane == 0 && q < O) gbo[q] = (float)s;
  } else if (q == GH_O) {
    point_loss_final(partial + (long)q * n_cta, n_cta, s, denom, rw, O, p1, p2, out2);
  }
}

// =============================================================================================
// Host side
// =============================================================================================
struct GenLayer {
  int I, Ipad, Kp;
  __nv_bfloat16 *hseq, *hseq_lo, *hmseq, *hmseq_lo, *in, *in_lo, *gates, *cst;
  __nv_bfloat16 *Wf, *Wf_lo, *Ub, *Wb;
  float *biasp, *bn;
  CUtensorMap tm_h, tm_h_lo, tm_hm, tm_hm_lo, tm_in, tm_in_lo, tm_wf, tm_wf_lo, tm_ub, tm_wb;   // K-major (recurrence, dx)
  CUtensorMap tm_hA_mn, tm_in_mn;                                                       // MN-major (weight gradients)
};

struct GenImpl {
  unsigned int* gbar = nullptr;         // grid-barrier counters of the persistent step launches (GBAR_N, zeroed per call)
  int gbar_next = 0;
  cudaStream_t side = nullptr;          // second half of the batch in the backward recurrence (see gen_backward)
  cudaEvent_t ev_fork = nullptr, ev_join = nullptr;
  int maxB = 0, Bp = 0, NRT = 0, T = 0, F = 0, O = 0, H = 0, L = 0, NB16 = 0;
  bool x3 = false, train_ws = false, gru = false, uq = false;
  std::vector<GenLayer> layers;
  __nv_bfloat16 *head_in = nullptr, *head_in_lo = nullptr;      // in[L]
  CUtensorMap tm_head_in;
  // tensor-core head (bf16): packed Wo (uq: [Wo | Wv], 32 rows), bf16 dLoss/dpred rows, per-tile loss partials
  __nv_bfloat16 *WoT = nullptr, *WoS = nullptr, *dpb = nullptr;
  float* head_tc_part = nullptr;
  CUtensorMap tm_wot, tm_wos, tm_dpb, tm_dpb_mn, tm_head_in_mn;
  float *cstate = nullptr, *dcstate = nullptr;
  __nv_bfloat16 *dz = nullptr, *dy = nullptr, *dhout = nullptr;
  CUtensorMap tm_dz, tm_dz_mn;
  float *bn_part = nullptr, *cs_part = nullptr;
  float* wg_part = nullptr;
  size_t wg_part_elems = 0;
  int head_ctas = 0, bn_ctas_max = 0, cs_chunks = 0;
  int BNU = 128;      // hidden units per backward tile
};

bool gen_supported(const lfmq_config& c, char* why, size_t n) {
  if (c.rnn_cell != LFMQ_CELL_LSTM && !c.forward_only) {
    snprintf(why, n, "training on the tensor-core paths is built for the LSTM cell only (GRU handles must be forward_only)");
    return false;
  }
  if (c.uq && !c.forward_only) {
    snprintf(why, n,
             "training on the tensor-core paths is built for the point-estimate head only (uq handles must be forward_only)");
    return false;
  }
  if (c.num_hidden % 64 != 0 || c.num_hidden > 512) {
    snprintf(why, n, "num_hidden must be a multiple of 64 and <= 512 (got %d)", c.num_hidden);
    return false;
  }
  if (c.n_outputs > GH_O) { snprintf(why, n, "n_outputs must be <= 16 (got %d)", c.n_outputs); return false; }
  if (c.n_inputs > 1024) { snprintf(why, n, "n_inputs must be <= 1024 (got %d)", c.n_inputs); return false; }
  if (c.precision == LFMQ_PREC_BF16X3 && !c.forward_only) {
    snprintf(why, n, "LFMQ_PREC_BF16X3 (fp32-tolerance forward) is built for forward_only handles");
    return false;
  }
  return true;
}

// Dropout and recurrent dropout are active in training and, on uq handles, always (MC dropout: `training=True` is a
// literal in rnn_uq_range_estimate.py:86,88), as on the fp32 path.
static bool gen_stochastic(const lfmq_config& c) { return c.train || c.uq; }

void gen_layout(TcState& st, const lfmq_config& c, const ParamLayout& pl, Carver& cv) {
  if (!st.gen) st.gen = new GenImpl;
  GenImpl& m = *st.gen;
  m.maxB = c.max_batch; m.T = c.seq_len; m.F = c.n_inputs; m.O = c.n_outputs; m.H = c.num_hidden; m.L = c.num_layers;
  m.Bp = (c.max_batch + 127) / 128 * 128;
  m.NRT = m.Bp / 128;
  m.NB16 = m.H / 16;
  m.x3 = c.precision == LFMQ_PREC_BF16X3;
  m.train_ws = !c.forward_only;
  m.gru = c.rnn_cell == LFMQ_CELL_GRU;
  m.uq = c.uq != 0;
  m.BNU = (m.H % 128 == 0) ? 128 : 64;
  const size_t T = m.T, Bp = m.Bp, H = m.H;
  const bool rec = (gen_stochastic(c) && c.recurrent_dropout > 0.f);
  m.layers.assign(m.L, GenLayer{});
  for (int l = 0; l < m.L; ++l) {
    GenLayer& ly = m.layers[l];
    ly.I = pl.layers[l].I;
    ly.Ipad = (ly.I + 63) / 64 * 64;
    ly.Kp = (int)H + ly.Ipad;
    ly.hseq = cv.take<__nv_bfloat16>((T + 1) * Bp * H);
    ly.hseq_lo = m.x3 ? cv.take<__nv_bfloat16>((T + 1) * Bp * H) : nullptr;
    ly.hmseq = rec ? cv.take<__nv_bfloat16>((T + 1) * Bp * H) : nullptr;
    ly.hmseq_lo = (rec && m.x3) ? cv.take<__nv_bfloat16>((T + 1) * Bp * H) : nullptr;
    ly.in = cv.take<__nv_bfloat16>(T * Bp * ly.Ipad);
    ly.in_lo = m.x3 ? cv.take<__nv_bfloat16>(T * Bp * ly.Ipad) : nullptr;
    ly.Wf = cv.take<__nv_bfloat16>((size_t)4 * H * ly.Kp);
    ly.Wf_lo = m.x3 ? cv.take<__nv_bfloat16>((size_t)4 * H * ly.Kp) : nullptr;
    ly.biasp = cv.take<float>(4 * H);
    ly.bn = cv.take<float>(4 * H);
    if (m.train_ws) {
      ly.gates = cv.take<__nv_bfloat16>(T * Bp * 4 * H);
      ly.cst = cv.take<__nv_bfloat16>(T * Bp * H);
      ly.Ub = cv.take<__nv_bfloat16>(H * 4 * H);
      ly.Wb = (l > 0) ? cv.take<__nv_bfloat16>((size_t)ly.I * 4 * H) : nullptr;
    } else {
      ly.gates = ly.cst = ly.Ub = ly.Wb = nullptr;
    }
  }
  m.head_in = cv.take<__nv_bfloat16>(T * Bp * H);
  m.head_in_lo = m.x3 ? cv.take<__nv_bfloat16>(T * Bp * H) : nullptr;
  m.WoT = cv.take<__nv_bfloat16>((m.uq ? 32 : 16) * H);
  m.WoS = cv.take<__nv_bfloat16>(H * 64);
  m.head_tc_part = cv.take<float>((size_t)GH_PART * T * m.NRT);
  m.dpb = m.train_ws ? cv.take<__nv_bfloat16>(T * Bp * 64) : nullptr;
  m.cstate = cv.take<float>(Bp * H);
  m.head_ctas = device_sm_count();
  if (m.train_ws) {
    m.dcstate = cv.take<float>(Bp * H);
    m.dz = cv.take<__nv_bfloat16>(T * Bp * 4 * H);
    m.dy = cv.take<__nv_bfloat16>(T * Bp * H);
    m.dhout = cv.take<__nv_bfloat16>(T * Bp * H);
    m.bn_ctas_max = (int)cdivl((long)T * m.maxB, GBN_ROWS);
    m.bn_part = cv.take<float>((size_t)2 * H * m.bn_ctas_max);
    m.cs_chunks = 1024;
    m.cs_part = cv.take<float>((size_t)4 * H * m.cs_chunks);
    const size_t Mmax = (H > 64 ? H : 128);               // dU: H rows; dW: Ipad rows (<= max(H, 64..1024))
    size_t mp = (Mmax + 255) / 256 * 256;
    for (int l = 0; l < m.L; ++l) {
      const size_t ip = ((size_t)m.layers[l].Ipad + 255) / 256 * 256;
      if (ip > mp) mp = ip;
    }
    m.wg_part_elems = (size_t)8 * mp * 4 * H;             // up to 8 K-splits
    m.wg_part = cv.take<float>(m.wg_part_elems);
  }
}

int gen_init(TcState& st, const lfmq_config& c) {
  GenImpl& m = *st.gen;
  const size_t T = m.T, Bp = m.Bp, H = m.H;
  int rc;
  for (int l = 0; l < m.L; ++l) {
    GenLayer& ly = m.layers[l];
    // every buffer that is an operand of a GEMM over padded rows / columns must hold finite values everywhere
    LFMQ_CUDA_CHECK(cudaMemset(ly.hseq, 0, (T + 1) * Bp * H * 2));
    if (ly.hseq_lo) LFMQ_CUDA_CHECK(cudaMemset(ly.hseq_lo, 0, (T + 1) * Bp * H * 2));
    if (ly.hmseq) LFMQ_CUDA_CHECK(cudaMemset(ly.hmseq, 0, (T + 1) * Bp * H * 2));
    if (ly.hmseq_lo) LFMQ_CUDA_CHECK(cudaMemset(ly.hmseq_lo, 0, (T + 1) * Bp * H * 2));
    LFMQ_CUDA_CHECK(cudaMemset(ly.in, 0, T * Bp * ly.Ipad * 2));
    if (ly.in_lo) LFMQ_CUDA_CHECK(cudaMemset(ly.in_lo, 0, T * Bp * ly.Ipad * 2));
    const uint64_t hrows = (T + 1) * Bp;
    if ((rc = gmap_2d(&ly.tm_h, ly.hseq, H, hrows, 64, 128))) return rc;
    if (ly.hseq_lo && (rc = gmap_2d(&ly.tm_h_lo, ly.hseq_lo, H, hrows, 64, 128))) return rc;
    if (ly.hmseq && (rc = gmap_2d(&ly.tm_hm, ly.hmseq, H, hrows, 64, 128))) return rc;
    if (ly.hmseq_lo && (rc = gmap_2d(&ly.tm_hm_lo, ly.hmseq_lo, H, hrows, 64, 128))) return rc;
    if ((rc = gmap_2d(&ly.tm_in, ly.in, ly.Ipad, T * Bp, 64, 128))) return rc;
    if (ly.in_lo && (rc = gmap_2d(&ly.tm_in_lo, ly.in_lo, ly.Ipad, T * Bp, 64, 128))) return rc;
    if ((rc = gmap_2d(&ly.tm_wf, ly.Wf, ly.Kp, 4 * H, 64, 256))) return rc;
    if (ly.Wf_lo && (rc = gmap_2d(&ly.tm_wf_lo, ly.Wf_lo, ly.Kp, 4 * H, 64, 256))) return rc;
    if (m.train_ws) {
      if ((rc = gmap_2d(&ly.tm_ub, ly.Ub, 4 * H, H, 64, m.BNU))) return rc;
      if (ly.Wb && (rc = gmap_2d(&ly.tm_wb, ly.Wb, 4 * H, ly.I, 64, (H % 128 == 0) ? 128 : 64))) return rc;
      // MN-major views for the weight gradients: slots 0..T-1 of (hmseq | hseq) against dz, boxes 64 (M) x 64 (rows)
      if ((rc = gmap_2d(&ly.tm_hA_mn, ly.hmseq ? ly.hmseq : ly.hseq, H, T * Bp, 64, 64))) return rc;
      if ((rc = gmap_2d(&ly.tm_in_mn, ly.in, ly.Ipad, T * Bp, 64, 64))) return rc;
    }
  }
  LFMQ_CUDA_CHECK(cudaMemset(m.head_in, 0, T * Bp * H * 2));
  if (m.head_in_lo) LFMQ_CUDA_CHECK(cudaMemset(m.head_in_lo, 0, T * Bp * H * 2));
  if ((rc = gmap_2d(&m.tm_head_in, m.head_in, H, T * Bp, 64, 128))) return rc;
  if ((rc = gmap_2d(&m.tm_wot, m.WoT, H, m.uq ? 32 : 16, 64, m.uq ? 32 : 16))) return rc;
  if (m.train_ws) {
    LFMQ_CUDA_CHECK(cudaMemset(m.dpb, 0, T * Bp * 64 * 2));       // columns >= 16 stay zero for good
    if ((rc = gmap_2d(&m.tm_wos, m.WoS, 64, H, 64, (H % 128 == 0) ? 128 : 64))) return rc;
    if ((rc = gmap_2d(&m.tm_dpb, m.dpb, 64, T * Bp, 64, 128))) return rc;
    if ((rc = gmap_2d(&m.tm_dpb_mn, m.dpb, 64, T * Bp, 64, 64))) return rc;
    if ((rc = gmap_2d(&m.tm_head_in_mn, m.head_in, H, T * Bp, 64, 64))) return rc;
  }
  if (m.train_ws) {
    LFMQ_CUDA_CHECK(cudaMemset(m.dz, 0, T * Bp * 4 * H * 2));
    LFMQ_CUDA_CHECK(cudaMemset(m.dy, 0, T * Bp * H * 2));
    LFMQ_CUDA_CHECK(cudaMemset(m.dhout, 0, T * Bp * H * 2));
    if ((rc = gmap_2d(&m.tm_dz, m.dz, 4 * H, T * Bp, 64, 128))) return rc;
    if ((rc = gmap_2d(&m.tm_dz_mn, m.dz, 4 * H, T * Bp, 64, 64))) return rc;
  }
#define LFMQ_GEMM_ATTR(BN_, EPI_)                                                                              \
  LFMQ_CUDA_CHECK(cudaFuncSetAttribute(tile_gemm_kernel<BN_, EPI_>, cudaFuncAttributeMaxDynamicSharedMemorySize, \
                                       GSmem<BN_, EPI_>::TOTAL))
  LFMQ_GEMM_ATTR(256, EPI_FWD);
  LFMQ_GEMM_ATTR(256, EPI_FWD_ACC);
  LFMQ_GEMM_ATTR(128, EPI_BWD);
  LFMQ_GEMM_ATTR(64, EPI_BWD);
  LFMQ_GEMM_ATTR(256, EPI_GRU_FWD);
  LFMQ_GEMM_ATTR(256, EPI_GRU_FWD_ACC);
  LFMQ_GEMM_ATTR(16, EPI_HEAD);
  LFMQ_GEMM_ATTR(32, EPI_HEAD_UQ);
  LFMQ_GEMM_ATTR(128, EPI_STORE);
  LFMQ_GEMM_ATTR(64, EPI_STORE);
#undef LFMQ_GEMM_ATTR
  if ((rc = wgrad_gemm_init())) return rc;
  const int hsmem = (int)((H / 64) * 16384 + H * GH_O * 4 + 64 + 1024);
  LFMQ_CUDA_CHECK(cudaFuncSetAttribute(ghead_rows_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, hsmem));
  if (m.train_ws) {
    const int bsm = (256 / ((int)H / 8) > 0 ? 256 / ((int)H / 8) : 1) * 2 * (int)H * 4;
    LFMQ_CUDA_CHECK(cudaFuncSetAttribute(gbn_drop_bwd_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, bsm));
  }
  LFMQ_CUDA_CHECK(cudaMalloc(&m.gbar, GBAR_N * sizeof(unsigned int)));
  LFMQ_CUDA_CHECK(cudaMemset(m.gbar, 0, GBAR_N * sizeof(unsigned int)));
  st.weights_dirty = 1;
  return 0;
}

// Persistent step launches need every CTA of the launch(es) running at once (they meet at a grid-wide barrier).
// `n_concurrent` launches of `ctas` CTAs each, `per_sm` resident CTAs of that instantiation per SM, within the handle's
// device share (persistent_cta_budget).  LFMQ_GEN_PERSIST=0 turns the mode off (one launch per time step, chained with
// programmatic dependent launch).
static bool gen_can_persist(const TcState& st, long ctas, int n_concurrent, int per_sm, int n_steps) {
  static const bool on = !(getenv("LFMQ_GEN_PERSIST") && atoi(getenv("LFMQ_GEN_PERSIST")) == 0);
  const GenImpl& m = *st.gen;
  return on && n_steps > 1 && m.gbar != nullptr &&
         ctas * n_concurrent <= persistent_cta_budget(device_sm_count(), per_sm, st.share_num, st.share_den) &&
         m.gbar_next + ctas * n_concurrent <= GBAR_N;
}

void gen_destroy(TcState& st) {
  if (st.gen && st.gen->side) {
    cudaStreamSynchronize(st.gen->side);
    cudaEventDestroy(st.gen->ev_fork);
    cudaEventDestroy(st.gen->ev_join);
    cudaStreamDestroy(st.gen->side);
  }
  if (st.gen && st.gen->gbar) cudaFree(st.gen->gbar);
  delete st.gen;
  st.gen = nullptr;
}

// Launch of one tile_gemm_kernel instantiation; `pdl`: with the programmatic-stream-serialization attribute.  The kernel
// loads weight tiles before its pdl_sync(), so a step may only overlap a predecessor that does not write them.
template <int BN, int EPI>
static int launch_tile_gemm(dim3 grid, cudaStream_t s, bool pdl, const GArgs& g, const EpiParams& ep, const CUtensorMap& a0,
                            const CUtensorMap& a1, const CUtensorMap& a2, const CUtensorMap& a3, const CUtensorMap& b0,
                            const CUtensorMap& b1) {
  return launch_pdl(tile_gemm_kernel<BN, EPI>, grid, dim3(GSmem<BN, EPI>::THREADS), GSmem<BN, EPI>::TOTAL, s, 1, pdl, g, ep,
                    a0, a1, a2, a3, b0, b1);
}

static int gen_pack(TcState& st, const ParamLayout& pl, const float* params, float eps, cudaStream_t s) {
  GenImpl& m = *st.gen;
  if (!st.weights_dirty) return 0;
  for (int l = 0; l < m.L; ++l) {
    GenLayer& ly = m.layers[l];
    const ParamLayout::Layer& o = pl.layers[l];
    GPackArgs a;
    a.H = m.H; a.I = ly.I; a.Ipad = ly.Ipad; a.Kp = ly.Kp; a.gru = m.gru ? 1 : 0;
    a.hs = m.x3 ? 1.0f : 0.5f;
    a.eps = eps;
    a.W = params + o.oW; a.U = params + o.oU; a.bias = params + o.ob;
    a.gamma = params + o.ogamma; a.beta = params + o.obeta; a.mean = params + o.omean; a.var = params + o.ovar;
    a.Wf = ly.Wf; a.Wf_lo = ly.Wf_lo; a.Ub = ly.Ub; a.Wb = ly.Wb; a.biasp = ly.biasp; a.bn = ly.bn;
    const long n = (long)4 * m.H * ly.Kp;
    gpack_kernel<<<(int)cdivl(n, 256), 256, 0, s>>>(a);
    LFMQ_LAUNCH_CHECK();
  }
  gpack_head_kernel<<<(int)cdivl((long)m.H * 64, 256), 256, 0, s>>>(m.H, m.O, params + pl.oWo, m.WoT, m.WoS);
  LFMQ_LAUNCH_CHECK();
  if (m.uq) {
    gpack_head_kernel<<<(int)cdivl((long)m.H * 16, 256), 256, 0, s>>>(m.H, m.O, params + pl.oWv, m.WoT + 16 * m.H, nullptr);
    LFMQ_LAUNCH_CHECK();
  }
  st.weights_dirty = 0;
  return 0;
}

// all layers' recurrences + BN/Dropout; leaves in[L] (the head input)
static int gen_run_trunk(TcState& st, const lfmq_config& c, const float* params, const float* x, int B, int64_t row0,
                         int64_t step, bool save, cudaStream_t s) {
  GenImpl& m = *st.gen;
  const int T = m.T, H = m.H, Bp = m.Bp;
  const int nrt = (B + 127) / 128;
  const bool rec = gen_stochastic(c) && c.recurrent_dropout > 0.f;
  const bool drop = gen_stochastic(c) && c.dropout > 0.f;
  LFMQ_CUDA_CHECK(cudaMemsetAsync(m.gbar, 0, GBAR_N * sizeof(unsigned int), s));
  m.gbar_next = 0;
  {
    const GenLayer& l0 = m.layers[0];
    const long n = (long)B * T * (l0.Ipad / 8);
    gcast_x_kernel<<<(int)cdivl(n, 256), 256, 0, s>>>(B, T, m.F, Bp, l0.Ipad, x, l0.in, l0.in_lo,
                                                      (save && !m.x3 && l0.Ipad > m.F) ? 1 : 0);
    LFMQ_LAUNCH_CHECK();
  }
  for (int l = 0; l < m.L; ++l) {
    GenLayer& ly = m.layers[l];
    EpiParams ep = {};
    ep.T = T; ep.B = B; ep.Bp = Bp; ep.H = H; ep.NRT = m.NRT; ep.NB16 = m.NB16; ep.row0 = row0;
    ep.bias = ly.biasp; ep.cstate = m.cstate; ep.hseq = ly.hseq; ep.hseq_lo = ly.hseq_lo;
    ep.hmseq = rec ? ly.hmseq : nullptr;
    ep.hmseq_lo = rec ? ly.hmseq_lo : nullptr;
    ep.gates = save ? ly.gates : nullptr;
    ep.cst = save ? ly.cst : nullptr;
    ep.accurate = m.x3 ? 1 : 0;
    ep.use_rec = rec ? 1 : 0;
    ep.rkey = dropout_key(c.seed, st.stream_base + 2 * l + 1, step, c.recurrent_dropout);
    const CUtensorMap& th = rec ? ly.tm_hm : ly.tm_h;
    const CUtensorMap& th_lo = rec ? ly.tm_hm_lo : ly.tm_h_lo;     // bf16x3
    // steps 1 .. T-1 as ONE persistent launch when all its CTAs fit on the machine at once (see GArgs::n_steps)
    const long fwd_ctas = (long)nrt * (4 * H / 256);
    const bool persist = gen_can_persist(st, fwd_ctas, 1, GSmem<256, EPI_FWD>::CTAS_PER_SM, T - 1);
    for (int t = 0; t < T; ++t) {
      ep.t = t;
      GArgs g = {};
      g.a_row_base = t * Bp;
      g.b_row_base = 0;
      if (persist && t == 1) {
        g.n_steps = T - 1;
        g.row_step = Bp;
        g.t_step = 1;
        g.gbar = m.gbar + m.gbar_next;
        m.gbar_next += nrt;
      }
      const int nkb_h = (t > 0) ? H / 64 : 0, nkb_x = ly.Ipad / 64;
      int ns = 0;
      // maps: A0 = h (or masked h), A1 = input, A2 = h low halves, A3 = input low halves; B0 = weights, B1 = their low halves
      if (nkb_h) g.seg[ns++] = GSeg{0, 0, nkb_h, 0, 0};
      g.seg[ns++] = GSeg{1, 0, nkb_x, 0, H};
      if (m.x3) {
        if (nkb_h) g.seg[ns++] = GSeg{2, 0, nkb_h, 0, 0};      // lo(h) hi(W)
        g.seg[ns++] = GSeg{3, 0, nkb_x, 0, H};
        if (nkb_h) g.seg[ns++] = GSeg{0, 1, nkb_h, 0, 0};      // hi(h) lo(W)
        g.seg[ns++] = GSeg{1, 1, nkb_x, 0, H};
      }
      g.n_seg = ns;
      // Steps after the first of a layer follow another step kernel: PDL.
      int rc;
#define LFMQ_FWD_LAUNCH(EPI_)                                                                                     \
  rc = launch_tile_gemm<256, EPI_>(dim3(nrt, 4 * H / 256), s, t > 0, g, ep, th, ly.tm_in, m.x3 ? th_lo : th,  \
                                   m.x3 ? ly.tm_in_lo : ly.tm_in, ly.tm_wf, m.x3 ? ly.tm_wf_lo : ly.tm_wf)
      if (m.gru && m.x3)
        LFMQ_FWD_LAUNCH(EPI_GRU_FWD_ACC);
      else if (m.gru)
        LFMQ_FWD_LAUNCH(EPI_GRU_FWD);
      else if (m.x3)
        LFMQ_FWD_LAUNCH(EPI_FWD_ACC);
      else
        LFMQ_FWD_LAUNCH(EPI_FWD);
#undef LFMQ_FWD_LAUNCH
      if (rc) return rc;
      if (persist && t == 1) break;              // that launch ran steps 1 .. T-1
    }
    const bool last = (l == m.L - 1);
    __nv_bfloat16* yo = last ? m.head_in : m.layers[l + 1].in;
    __nv_bfloat16* yo_lo = last ? m.head_in_lo : m.layers[l + 1].in_lo;
    const long n = (long)T * B * (H / 8);
    gbn_drop_fwd_kernel<<<(int)cdivl(n, 256), 256, 0, s>>>(B, T, H, Bp, ly.hseq, ly.hseq_lo, ly.bn, drop ? 1 : 0,
                                                           dropout_key(c.seed, st.stream_base + 2 * l, step, c.dropout), row0, yo, yo_lo);
    LFMQ_LAUNCH_CHECK();
  }
  return 0;
}

// `db` (nullable): row Mvalid of the product (A's constant-one column, see gcast_x_kernel) = colsum(dz)
static int gen_wgrad(GenImpl& m, const CUtensorMap& tm_a, int Mvalid, float* dst, cudaStream_t s, float* db = nullptr) {
  const int Ntot = 4 * m.H;
  int S = 0, Mpad = 0, rc;
  if ((rc = wgrad_gemm(tm_a, m.tm_dz_mn, (long)m.T * m.Bp, db ? Mvalid + 1 : Mvalid, Ntot, m.wg_part, m.wg_part_elems,
                       false, s, &S, &Mpad)))
    return rc;
  const long n4 = (long)Mvalid * Ntot / 4;
  gwgrad_reduce_kernel<<<(int)cdivl(n4, 256), 256, 0, s>>>(S, Mvalid, Mpad, Ntot, m.wg_part, dst, 0);
  LFMQ_LAUNCH_CHECK();
  if (db) {
    gwgrad_reduce_kernel<<<(int)cdivl(Ntot / 4, 256), 256, 0, s>>>(S, 1, Mpad, Ntot, m.wg_part, db, Mvalid);
    LFMQ_LAUNCH_CHECK();
  }
  return 0;
}

static int gen_run_head(TcState& st, const lfmq_config& c, const ParamLayout& pl, const float* params, float* grads,
                        const float* y, int B, const float* denom, float* preds, float* out2, bool train,
                        cudaStream_t s) {
  GenImpl& m = *st.gen;
  if (m.x3) {
    // LFMQ_PREC_BF16X3 (1e-4 tolerance): the fp32-accumulating SIMT head.  Its handles are forward-only, so it predicts.
    GHeadParams h = {};
    h.B = B; h.T = m.T; h.O = m.O; h.H = m.H; h.Bp = m.Bp; h.NRT = (B + 127) / 128;
    h.Wo = params + pl.oWo; h.bo = params + pl.obo;
    h.preds = preds;
    h.yin_lo = m.head_in_lo;
    int grid = m.T * h.NRT;
    if (grid > m.head_ctas) grid = m.head_ctas;
    const int hsmem = (m.H / 64) * 16384 + m.H * GH_O * 4 + 64 + 1024;
    ghead_rows_kernel<<<grid, 128, hsmem, s>>>(h, m.tm_head_in);
    LFMQ_LAUNCH_CHECK();
    return 0;
  }
  // Tensor-core head: pred = y Wo as a wgmma GEMM (N = 16) with the loss in its epilogue; training adds
  // dy = dpred Wo^T (K = 16 padded to one k-block) and dWo = y^T dpred (the weight-gradient GEMM, N padded to 256).
  const int ntile = m.T * m.NRT;                  // every row tile of the time-major buffers (zeros beyond the batch)
  EpiParams ep = {};
  ep.T = m.T; ep.B = B; ep.Bp = m.Bp; ep.H = m.H; ep.NRT = m.NRT; ep.NB16 = m.NB16;
  ep.hy = y; ep.hdenom = denom; ep.hrw = train ? st.row_w : nullptr; ep.hbo = params + pl.obo; ep.hpreds = preds; ep.hdpb = m.dpb;
  ep.hpartial = m.head_tc_part; ep.hp1 = c.target_lambda; ep.hp2 = c.rnn_lambda; ep.hO = m.O;
  ep.htarget = c.target_idx; ep.htrain = train ? 1 : 0;
  GArgs g = {};
  g.n_seg = 1;
  g.seg[0] = GSeg{0, 0, m.H / 64, 0, 0};
  int rc;
  if ((rc = launch_tile_gemm<16, EPI_HEAD>(dim3(ntile, 1), s, false, g, ep, m.tm_head_in, m.tm_head_in, m.tm_head_in,
                                              m.tm_head_in, m.tm_wot, m.tm_wot)))
    return rc;
  if (train) {
    EpiParams es = {};
    es.out = m.dy;
    es.ldc = m.H;
    es.Bp = m.Bp;
    GArgs gd = {};
    gd.n_seg = 1;
    gd.seg[0] = GSeg{0, 0, 1, 0, 0};
    const int row_tiles = m.T * m.Bp / 128;
    gd.lin_cols = (m.H % 128 == 0) ? m.H / 128 : m.H / 64;
    if (m.H % 128 == 0)
      rc = launch_tile_gemm<128, EPI_STORE>(dim3(row_tiles * (m.H / 128)), s, false, gd, es, m.tm_dpb, m.tm_dpb, m.tm_dpb,
                                               m.tm_dpb, m.tm_wos, m.tm_wos);
    else
      rc = launch_tile_gemm<64, EPI_STORE>(dim3(row_tiles * (m.H / 64)), s, false, gd, es, m.tm_dpb, m.tm_dpb, m.tm_dpb,
                                              m.tm_dpb, m.tm_wos, m.tm_wos);
    if (rc) return rc;
    int S = 0, Mpad = 0;
    if ((rc = wgrad_gemm(m.tm_head_in_mn, m.tm_dpb_mn, (long)m.T * m.Bp, m.H, 256, m.wg_part, m.wg_part_elems, false, s,
                         &S, &Mpad)))
      return rc;
    ghead_wo_reduce_kernel<<<(m.H * m.O + 255) / 256, 256, 0, s>>>(S, m.H, m.O, Mpad, m.wg_part, grads + pl.oWo);
    LFMQ_LAUNCH_CHECK();
  }
  if (y) {
    ghead_reduce_kernel<<<(GH_PART * 32 + 255) / 256, 256, 0, s>>>(ntile, m.head_tc_part, m.O, denom, ep.hrw,
                                                                  c.target_lambda,
                                                                  c.rnn_lambda, train ? 1 : 0,
                                                                  grads ? grads + pl.obo : nullptr, out2);
    LFMQ_LAUNCH_CHECK();
  }
  return 0;
}

int gen_forward(TcState& st, const lfmq_config& c, const ParamLayout& pl, const float* params, const float* x, int B,
                int64_t row0, int64_t step, float* preds, cudaStream_t s) {
  int rc;
  if ((rc = gen_pack(st, pl, params, c.bn_epsilon, s))) return rc;
  st.prof->begin(LFMQ_REGION_FWD, s);
  if ((rc = gen_run_trunk(st, c, params, x, B, row0, step, false, s))) return rc;
  st.prof->end(LFMQ_REGION_FWD, s);
  st.prof->begin(LFMQ_REGION_HEAD, s);
  if ((rc = gen_run_head(st, c, pl, params, nullptr, nullptr, B, nullptr, preds, nullptr, false, s))) return rc;
  st.prof->end(LFMQ_REGION_HEAD, s);
  return 0;
}

// The two heads of a uq handle on y = in[L]: bf16, one N = 32 GEMM over [Wo | Wv]; bf16x3, the fp32-accumulating SIMT
// head once per head.
static int gen_run_head_uq(GenImpl& m, const ParamLayout& pl, const float* params, int B, float* preds, float* var,
                           cudaStream_t s) {
  if (m.x3) {
    GHeadParams h = {};
    h.B = B; h.T = m.T; h.O = m.O; h.H = m.H; h.Bp = m.Bp; h.NRT = (B + 127) / 128;
    h.yin_lo = m.head_in_lo;
    int grid = m.T * h.NRT;
    if (grid > m.head_ctas) grid = m.head_ctas;
    const int hsmem = (m.H / 64) * 16384 + m.H * GH_O * 4 + 64 + 1024;
    for (int v = 0; v < 2; ++v) {
      h.Wo = params + (v ? pl.oWv : pl.oWo);
      h.bo = params + (v ? pl.obv : pl.obo);
      h.preds = v ? var : preds;
      h.softplus_floor = v;
      ghead_rows_kernel<<<grid, 128, hsmem, s>>>(h, m.tm_head_in);
      LFMQ_LAUNCH_CHECK();
    }
    return 0;
  }
  EpiParams ep = {};
  ep.T = m.T; ep.B = B; ep.Bp = m.Bp; ep.H = m.H; ep.NRT = m.NRT; ep.NB16 = m.NB16;
  ep.hbo = params + pl.obo; ep.hpreds = preds; ep.hO = m.O;
  ep.hbv = params + pl.obv; ep.hvar = var;
  GArgs g = {};
  g.n_seg = 1;
  g.seg[0] = GSeg{0, 0, m.H / 64, 0, 0};
  return launch_tile_gemm<32, EPI_HEAD_UQ>(dim3(m.T * m.NRT, 1), s, false, g, ep, m.tm_head_in, m.tm_head_in,
                                           m.tm_head_in, m.tm_head_in, m.tm_wot, m.tm_wot);
}

int gen_forward_uq(TcState& st, const lfmq_config& c, const ParamLayout& pl, const float* params, const float* x,
                   int B, int64_t row0, int64_t step, float* preds, float* var, cudaStream_t s) {
  int rc;
  if ((rc = gen_pack(st, pl, params, c.bn_epsilon, s))) return rc;
  st.prof->begin(LFMQ_REGION_FWD, s);
  if ((rc = gen_run_trunk(st, c, params, x, B, row0, step, false, s))) return rc;
  st.prof->end(LFMQ_REGION_FWD, s);
  st.prof->begin(LFMQ_REGION_HEAD, s);
  if ((rc = gen_run_head_uq(*st.gen, pl, params, B, preds, var, s))) return rc;
  st.prof->end(LFMQ_REGION_HEAD, s);
  return 0;
}

int gen_backward(TcState& st, const lfmq_config& c, const ParamLayout& pl, const float* params, float* grads,
                 const float* x, const float* y, int B, int64_t row0, int64_t step, const float* denom, float* tail,
                 cudaStream_t s) {
  GenImpl& m = *st.gen;
  const int T = m.T, H = m.H, Bp = m.Bp;
  const int nrt = (B + 127) / 128;
  const bool rec = c.train && c.recurrent_dropout > 0.f;
  const bool drop = c.train && c.dropout > 0.f;
  int rc;
  if ((rc = gen_pack(st, pl, params, c.bn_epsilon, s))) return rc;
  st.prof->begin(LFMQ_REGION_FWD, s);
  if ((rc = gen_run_trunk(st, c, params, x, B, row0, step, true, s))) return rc;
  st.prof->end(LFMQ_REGION_FWD, s);
  if (nrt < m.NRT) {
    // a smaller batch than an earlier call on this handle: the weight-gradient GEMMs sum over all T*Bp time-major rows,
    // so the rows of the row tiles that are not launched now must be zero (they may hold an earlier call's values)
    const size_t tail_rows = (size_t)(Bp - nrt * 128);
    LFMQ_CUDA_CHECK(cudaMemset2DAsync(m.dz + (size_t)nrt * 128 * 4 * H, (size_t)Bp * 4 * H * 2, 0, tail_rows * 4 * H * 2, T, s));
  }
  st.prof->begin(LFMQ_REGION_HEAD, s);
  if ((rc = gen_run_head(st, c, pl, params, grads, y, B, denom, nullptr, tail, true, s))) return rc;
  st.prof->end(LFMQ_REGION_HEAD, s);
  for (int l = m.L - 1; l >= 0; --l) {
    GenLayer& ly = m.layers[l];
    const ParamLayout::Layer& o = pl.layers[l];
    st.prof->begin(LFMQ_REGION_BWD, s);
    {   // Dropout / BN backward of this layer's output: dy -> dhout, dgamma, dbeta
      const int ctas = (int)cdivl((long)T * B, GBN_ROWS);
      const int RL = 256 / (H / 8) > 0 ? 256 / (H / 8) : 1;
      gbn_drop_bwd_kernel<<<ctas, 256, RL * 2 * H * 4, s>>>(B, T, H, Bp, m.dy, ly.hseq, ly.bn, drop ? 1 : 0,
                                                           dropout_key(c.seed, st.stream_base + 2 * l, step, c.dropout), row0, m.dhout, m.bn_part);
      LFMQ_LAUNCH_CHECK();
      gpartial_reduce_kernel<<<(2 * H * 32 + 255) / 256, 256, 0, s>>>(ctas, H, H, m.bn_part, grads + o.ogamma,
                                                                    grads + o.obeta);
      LFMQ_LAUNCH_CHECK();
    }
    EpiParams ep = {};
    ep.T = T; ep.B = B; ep.Bp = Bp; ep.H = H; ep.NRT = m.NRT; ep.NB16 = m.NB16; ep.row0 = row0;
    ep.gates = ly.gates; ep.cst = ly.cst; ep.dhout = m.dhout; ep.dcstate = m.dcstate; ep.dz = m.dz;
    ep.use_rec = rec ? 1 : 0;
    ep.rkey = dropout_key(c.seed, st.stream_base + 2 * l + 1, step, c.recurrent_dropout);
    // The step's epilogue is HBM-bound (saved gates / cell states in, dz out: ~46 MB per step at H = 512) and its
    // mainloop L2-bound, and one launch puts every CTA into the same phase at the same time.  Two half-batches on two
    // streams (each its own PDL chain) drift apart, so one half's epilogue runs beside the other's mainloop.
    const bool split = nrt >= 16;
    const int n_a = split ? (nrt + 1) / 2 : nrt, n_b = nrt - n_a;
    if (split) {
      if (!m.side) {
        LFMQ_CUDA_CHECK(cudaStreamCreateWithFlags(&m.side, cudaStreamNonBlocking));
        LFMQ_CUDA_CHECK(cudaEventCreateWithFlags(&m.ev_fork, cudaEventDisableTiming));
        LFMQ_CUDA_CHECK(cudaEventCreateWithFlags(&m.ev_join, cudaEventDisableTiming));
      }
      LFMQ_CUDA_CHECK(cudaEventRecord(m.ev_fork, s));
      LFMQ_CUDA_CHECK(cudaStreamWaitEvent(m.side, m.ev_fork, 0));
    }
    // steps T-2 .. 0 of each chain as ONE persistent launch when all CTAs of both chains fit on the machine at once
    const long bwd_ctas = (long)n_a * (H / m.BNU);
    const bool persist = gen_can_persist(st, bwd_ctas, split ? 2 : 1, 1, T - 1);
    for (int t = T - 1; t >= 0; --t) {
      for (int half = 0; half < (split ? 2 : 1); ++half) {       // launches interleaved: neither chain lags the other
        cudaStream_t hs = half ? m.side : s;
        const int rt_off = half ? n_a : 0, n_rt = half ? n_b : n_a;
        ep.t = t;
        ep.has_rec = (t < T - 1) ? 1 : 0;
        GArgs g = {};
        g.a_row_base = (t + 1) * Bp;      // dz_{t+1}
        g.b_row_base = 0;
        g.rt_off = rt_off;
        g.n_seg = ep.has_rec ? 1 : 0;
        g.seg[0] = GSeg{0, 0, 4 * H / 64, 0, 0};
        if (persist && t == T - 2) {
          g.n_steps = T - 1;
          g.row_step = -Bp;
          g.t_step = -1;
          g.gbar = m.gbar + m.gbar_next;
          m.gbar_next += n_rt;
        }
        if (m.BNU == 128)
          rc = launch_tile_gemm<128, EPI_BWD>(dim3(n_rt, H / 128), hs, t < T - 1, g, ep, m.tm_dz, m.tm_dz, m.tm_dz,
                                                 m.tm_dz, ly.tm_ub, ly.tm_ub);
        else
          rc = launch_tile_gemm<64, EPI_BWD>(dim3(n_rt, H / 64), hs, t < T - 1, g, ep, m.tm_dz, m.tm_dz, m.tm_dz,
                                                m.tm_dz, ly.tm_ub, ly.tm_ub);
        if (rc) return rc;
      }
      if (persist && t == T - 2) break;          // those launches ran steps T-2 .. 0
    }
    if (split) {
      LFMQ_CUDA_CHECK(cudaEventRecord(m.ev_join, m.side));
      LFMQ_CUDA_CHECK(cudaStreamWaitEvent(s, m.ev_join, 0));
    }
    st.prof->end(LFMQ_REGION_BWD, s);
    st.prof->begin(LFMQ_REGION_WGRAD, s);
    if ((rc = gen_wgrad(m, ly.tm_hA_mn, H, grads + o.oU, s))) return rc;
    // first layer: the input buffer's first padding column is constant one (gcast_x_kernel), so db falls out of the dW GEMM
    const bool ones_db = (l == 0) && !m.x3 && ly.Ipad > ly.I;
    if ((rc = gen_wgrad(m, ly.tm_in_mn, ly.I, grads + o.oW, s, ones_db ? grads + o.ob : nullptr))) return rc;
    if (!ones_db) {   // db = column sums of dz over the T*Bp rows (rows beyond the batch are zero)
      const long rows = (long)T * Bp;
      const long rpc = cdivl(rows, m.cs_chunks);
      gcolsum_kernel<<<dim3((4 * H / 8 + 127) / 128, m.cs_chunks), 128, 0, s>>>(rows, 4 * H, rpc, m.dz, m.cs_part);
      LFMQ_LAUNCH_CHECK();
      gpartial_reduce_kernel<<<(4 * H * 32 + 255) / 256, 256, 0, s>>>(m.cs_chunks, 4 * H, 0, m.cs_part,
                                                                    grads + o.ob, nullptr);
      LFMQ_LAUNCH_CHECK();
    }
    if (l > 0) {   // dLoss/dy_{l-1} = dz W^T  -> dy (bf16 [T*Bp][H])
      EpiParams es = {};
      es.out = m.dy;
      es.ldc = H;
      GArgs g = {};
      g.a_row_base = 0;
      g.b_row_base = 0;
      g.n_seg = 1;
      g.seg[0] = GSeg{0, 0, 4 * H / 64, 0, 0};
      const int row_tiles = T * Bp / 128;
      g.lin_cols = (H % 128 == 0) ? H / 128 : H / 64;
      if (H % 128 == 0)
        rc = launch_tile_gemm<128, EPI_STORE>(dim3(row_tiles * (H / 128)), s, false, g, es, m.tm_dz, m.tm_dz, m.tm_dz,
                                                 m.tm_dz, ly.tm_wb, ly.tm_wb);
      else
        rc = launch_tile_gemm<64, EPI_STORE>(dim3(row_tiles * (H / 64)), s, false, g, es, m.tm_dz, m.tm_dz, m.tm_dz,
                                                m.tm_dz, ly.tm_wb, ly.tm_wb);
      if (rc) return rc;
    }
    st.prof->end(LFMQ_REGION_WGRAD, s);
  }
  (void)x;
  return 0;
}

}  // namespace lfmq
