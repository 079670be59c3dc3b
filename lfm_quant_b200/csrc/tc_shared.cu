// Definitions of tc_shared.h: the bf16 tensor-map encoder and the weight-gradient GEMM of both tensor-core paths.
#include "tc_shared.h"

#include <cuda_bf16.h>

#include "sm90.cuh"

namespace lfmq {

using namespace sm90;

typedef CUresult (*PFN_encodeTiled)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                    const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                    CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

int encode_map_bf16(CUtensorMap* m, const void* base, int rank, const uint64_t* dims, const uint64_t* strides_bytes,
                    const uint32_t* box, CUtensorMapSwizzle sw) {
  static PFN_encodeTiled enc = nullptr;
  if (!enc) {
    void* fn = nullptr;
    cudaDriverEntryPointQueryResult q;
    LFMQ_CUDA_CHECK(cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &fn, cudaEnableDefault, &q));
    enc = reinterpret_cast<PFN_encodeTiled>(fn);
    if (!enc) {
      LFMQ_SET_ERR("cuTensorMapEncodeTiled not available");
      return LFMQ_ERR_CUDA;
    }
  }
  cuuint64_t d[5], st[4];
  cuuint32_t bx[5], es[5];
  for (int i = 0; i < rank; ++i) { d[i] = dims[i]; bx[i] = box[i]; es[i] = 1; }
  for (int i = 0; i + 1 < rank; ++i) st[i] = strides_bytes[i];
  CUresult r = enc(m, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, (cuuint32_t)rank, const_cast<void*>(base), d, st, bx, es,
                   CU_TENSOR_MAP_INTERLEAVE_NONE, sw, CU_TENSOR_MAP_L2_PROMOTION_L2_128B,
                   CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    LFMQ_SET_ERR("cuTensorMapEncodeTiled failed with %d (rank %d, dims %llu x %llu, box %u x %u)", (int)r, rank,
                 (unsigned long long)dims[0], (unsigned long long)dims[1], box[0], box[1]);
    return LFMQ_ERR_CUDA;
  }
  return 0;
}

// =============================================================================================
// Weight gradients: grid = (M tiles of 128, N tiles of 256, K splits); deterministic split-K through fp32 partials.
// =============================================================================================
struct WgradParams {
  int n_kblocks, kb_per_split, Mpad, Ntot;
  float* partial;       // [S][Mpad][Ntot]
};
struct WgradCfg {
  static constexpr int THREADS = 2 * 128 + 32;      // two consumer warpgroups (M rows 0-63 / 64-127) + TMA producer warp
  static constexpr uint32_t A_BYTES = 16384;
  static constexpr uint32_t STAGE_BYTES = A_BYTES + 32768;
  static constexpr int STAGES = (int)(196608u / STAGE_BYTES);
  static constexpr uint32_t SMEM = STAGES * STAGE_BYTES + 1024 + 256;
};

__global__ void __launch_bounds__(WgradCfg::THREADS, 1)
    wgrad_kernel(WgradParams p, const __grid_constant__ CUtensorMap tm_a, const __grid_constant__ CUtensorMap tm_b) {
  pdl_sync();
  using C = WgradCfg;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint64_t* full = reinterpret_cast<uint64_t*>(smem + C::STAGES * C::STAGE_BYTES);
  uint64_t* empty = full + C::STAGES;
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int m0 = blockIdx.x * 128, n0 = blockIdx.y * 256;
  const int kb_beg = blockIdx.z * p.kb_per_split;
  const int kb_end = min(p.n_kblocks, kb_beg + p.kb_per_split);
  const int nkb = max(0, kb_end - kb_beg);
  if (tid == 0) {
    for (int s = 0; s < C::STAGES; ++s) {
      mbar_init(&full[s], 1);
      mbar_init(&empty[s], 8);              // one arrive per consumer warp
    }
    fence_mbar_init();
  }
  __syncthreads();
  if (warp == 8) {
    if (lane == 0) {
      for (int i = 0; i < nkb; ++i) {
        const int s = i % C::STAGES;
        if (i >= C::STAGES) mbar_wait(&empty[s], ((i / C::STAGES) - 1) & 1);
        mbar_arrive_expect_tx(&full[s], C::STAGE_BYTES);
        uint8_t* st = smem + s * C::STAGE_BYTES;
        const int krow = (kb_beg + i) * 64;
        for (int mb = 0; mb < 2; ++mb) tma_load_2d(st + mb * 8192, &tm_a, &full[s], m0 + mb * 64, krow);
        for (int nb = 0; nb < 4; ++nb) tma_load_2d(st + C::A_BYTES + nb * 8192, &tm_b, &full[s], n0 + nb * 64, krow);
      }
    }
  } else {
    const int wg = warp >> 2, cq = lane & 3;
    float acc[128];
#pragma unroll
    for (int i = 0; i < 128; ++i) acc[i] = 0.f;
    for (int i = 0; i < nkb; ++i) {
      const int s = i % C::STAGES;
      mbar_wait(&full[s], (i / C::STAGES) & 1);
      uint8_t* st = smem + s * C::STAGE_BYTES;
      wgmma_fence();
#pragma unroll
      for (int k16 = 0; k16 < 4; ++k16) {
        const uint64_t db = make_smem_desc(smem_u32(st + C::A_BYTES) + k16 * 2048, 8192, 1024, LAYOUT_SW128);
        const uint64_t da = make_smem_desc(smem_u32(st + wg * 8192) + k16 * 2048, 8192, 1024, LAYOUT_SW128);
        wgmma_m64n256k16<1, 1>(acc, da, db, 1);
      }
      wgmma_commit();
      wgmma_wait<1>();                      // the previous stage's MMAs are complete: release it
      if (i > 0 && lane == 0) mbar_arrive(&empty[(i - 1) % C::STAGES]);
    }
    wgmma_wait<0>();
    fence_regs(acc);
    const int row = m0 + 64 * wg + 16 * (warp & 3) + (lane >> 2);
    float* out = p.partial + ((long)blockIdx.z * p.Mpad + row) * p.Ntot + n0 + 2 * cq;
#pragma unroll
    for (int i = 0; i < 128; i += 2)
      *reinterpret_cast<float2*>(out + (long)8 * ((i >> 1) & 1) * p.Ntot + 8 * (i >> 2)) = make_float2(acc[i], acc[i + 1]);
  }
}

int wgrad_gemm_init() {
  LFMQ_CUDA_CHECK(cudaFuncSetAttribute(wgrad_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, WgradCfg::SMEM));
  return 0;
}

int wgrad_gemm(const CUtensorMap& tm_a, const CUtensorMap& tm_b, long rows, int Mvalid, int Ntot, float* partial,
               size_t partial_elems, bool pdl, cudaStream_t s, int* S_out, int* Mpad_out) {
  const int mt = (Mvalid + 127) / 128;
  const int Mpad = mt * 128;
  WgradParams wp;
  wp.n_kblocks = (int)((rows + 63) / 64);
  // K splits: one wave of CTAs, within what the partial buffer holds
  int S = device_sm_count() / (mt * (Ntot / 256));
  const size_t smax = partial_elems / ((size_t)Mpad * Ntot);
  if ((size_t)S > smax) S = (int)smax;
  if (S > 64) S = 64;
  if (S < 1) S = 1;
  if (S > wp.n_kblocks) S = wp.n_kblocks;
  wp.kb_per_split = (wp.n_kblocks + S - 1) / S;
  S = (wp.n_kblocks + wp.kb_per_split - 1) / wp.kb_per_split;
  wp.Mpad = Mpad;
  wp.Ntot = Ntot;
  wp.partial = partial;
  if ((size_t)S * Mpad * Ntot > partial_elems) {
    LFMQ_SET_ERR("weight-gradient partial buffer too small");
    return LFMQ_ERR_WORKSPACE;
  }
  if (int rc = launch_pdl(wgrad_kernel, dim3(mt, Ntot / 256, S), dim3(WgradCfg::THREADS), WgradCfg::SMEM, s, 1, pdl, wp,
                          tm_a, tm_b))
    return rc;
  *S_out = S;
  *Mpad_out = Mpad;
  return 0;
}

}  // namespace lfmq
