// What the two tensor-core paths share: the handle's tensor-core state, the bf16 tensor-map encoder and the
// weight-gradient GEMM.  The cluster path is lstm_tc.cu, the general path rnn_tc.cu; both are defined in tc_shared.cu.
#pragma once
#include <cuda.h>

#include <vector>

#include "../../include/lfmq.h"
#include "common.cuh"

namespace lfmq {

struct TcImpl;
struct GenImpl;

// Where each tensor of a handle sits in its flat parameter vector, in floats (the gradient vector has the same layout
// over its trainable part).  layout() in lfmq_api.cu fills it with the parameter specs; every path reads it.
struct ParamLayout {
  struct Layer {
    int64_t oW, oU, ob, ogamma, obeta, omean, ovar;
    int I;                      // input width: n_inputs for layer 0, num_hidden above
  };
  std::vector<Layer> layers;    // none on a dense handle
  int64_t oWo = 0, obo = 0;     // OUTPUT_1, or OUTPUT_TARGET_1 on a uq handle
  int64_t oWv = -1, obv = -1;   // uq: OUTPUT_VARIANCE_1
};

// Tensor-core state of a handle.  layout() in lfmq_api.cu sets up at most one of the two paths.
struct TcState {
  int weights_dirty = 1;        // the parameters changed since the path last packed its bf16 copies of them
  int stream_base = 0;          // first Philox stream index of the handle's layers (stage s of a forecast chain: 2 (L0+s-1))
  int share_num = 1;            // lfmq_set_device_share: the fraction of the SMs this handle may count on for the
  int share_den = 1;            // co-residency of a persistent launch (persistent_cta_budget)
  Profiler* prof = nullptr;
  const float* row_w = nullptr; // lfmq_set_row_weights: the training batch's row weights, read by the head's loss
  TcImpl* impl = nullptr;       // cluster path
  GenImpl* gen = nullptr;       // general path
};

// The most CTAs a persistent launch (CTAs that wait for each other at a barrier in global memory) may have so that all of
// them are resident at once, given sm_count SMs, ctas_per_sm resident CTAs of its kernel on an otherwise empty SM and a
// device share num/den (0 < num <= den).  The whole device (num == den): sm_count * ctas_per_sm.  A share below one:
// floor(sm_count * num / den) CTAs, one per SM -- then every set of concurrent handles whose shares sum to at most one
// leaves an SM empty while any of their persistent launches still waits for a CTA (DESIGN.md section 6a).
inline long persistent_cta_budget(int sm_count, int ctas_per_sm, int num, int den) {
  if (num >= den) return (long)sm_count * ctas_per_sm;
  return (long)sm_count * num / den;
}

// bf16 tiled tensor map: dims and box innermost first, byte strides of dims 1 .. rank-1, no interleave, 128-byte L2
// promotion, no out-of-bounds fill.
int encode_map_bf16(CUtensorMap* m, const void* base, int rank, const uint64_t* dims, const uint64_t* strides_bytes,
                    const uint32_t* box, CUtensorMapSwizzle sw);

// The 2-D case: `outer` rows of `inner` elements, row_stride_bytes apart.
inline int encode_map_2d(CUtensorMap* m, const void* base, uint64_t inner, uint64_t outer, uint64_t row_stride_bytes,
                         uint32_t box_inner, uint32_t box_outer, CUtensorMapSwizzle sw) {
  const uint64_t dims[2] = {inner, outer};
  const uint32_t box[2] = {box_inner, box_outer};
  return encode_map_bf16(m, base, 2, dims, &row_stride_bytes, box, sw);
}

// Weight gradient D[Mvalid x Ntot] = A^T B over `rows` rows, both operands MN-major straight from their row-major
// buffers (maps with 64 x 64 SWIZZLE_128B boxes), Ntot a multiple of 256.  The rows are split S ways to fill the machine;
// the fp32 partials [S][Mpad][Ntot] go to `partial` (room for partial_elems floats) and the caller reduces them.
// `pdl`: launched with programmatic stream serialization (the kernel waits for its predecessor at entry).
// wgrad_gemm_init() sets the kernel's shared-memory limit on the current device; every path calls it in its init.
int wgrad_gemm_init();
int wgrad_gemm(const CUtensorMap& tm_a, const CUtensorMap& tm_b, long rows, int Mvalid, int Ntot, float* partial,
               size_t partial_elems, bool pdl, cudaStream_t s, int* S_out, int* Mpad_out);

}  // namespace lfmq
