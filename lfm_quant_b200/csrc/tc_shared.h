// What the two tensor-core paths share: the handle's tensor-core state, the bf16 tensor-map encoder and the
// weight-gradient GEMM.  The cluster path is lstm_tc.cu, the general path rnn_tc.cu; both are defined in tc_shared.cu.
#pragma once
#include <cuda.h>

#include "../../include/lfmq.h"
#include "common.cuh"

namespace lfmq {

struct TcImpl;
struct GenImpl;

// Tensor-core state of a handle.  layout() in lfmq_api.cu sets up at most one of the two paths.
struct TcState {
  int weights_dirty = 1;        // the parameters changed since the path last packed its bf16 copies of them
  Profiler* prof = nullptr;
  TcImpl* impl = nullptr;       // cluster path
  GenImpl* gen = nullptr;       // general path
};

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
