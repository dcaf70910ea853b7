// TMA (cp.async.bulk.tensor) + mbarrier helpers, sm_90a. Hand-written PTX wrappers; no CUTLASS.
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>

#include <cstdint>

#include "common.cuh"

namespace b200 {

// ---- host: tensor-map construction through the runtime's driver entry point (no -lcuda link) ----
using EncodeTiledFn = CUresult (*)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                   const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                   CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

inline EncodeTiledFn encodeTiled() {
  static EncodeTiledFn fn = [] {
    void*                            p = nullptr;
    cudaDriverEntryPointQueryResult q;
    cudaError_t e = cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q);
    if (e != cudaSuccess || q != cudaDriverEntryPointSuccess || !p)
      fail(B200MOL_ERR_CUDA, "cuTensorMapEncodeTiled entry point unavailable");
    return reinterpret_cast<EncodeTiledFn>(p);
  }();
  return fn;
}

// 2-D row-major tensor of 4-byte elements [rows][cols], box [boxRows][boxCols], swizzle chosen by box width.
// Returns the swizzle XOR mask for (offset>>7) (7 = 128B, 3 = 64B, 1 = 32B, 0 = none).
inline int makeTensorMap2D(CUtensorMap* tm, const void* base, uint64_t rows, uint64_t cols, uint32_t boxRows,
                           uint32_t boxCols, CUtensorMapDataType dt = CU_TENSOR_MAP_DATA_TYPE_UINT32,
                           uint32_t elemBytes = 4) {
  const uint32_t     innerBytes = boxCols * elemBytes;
  CUtensorMapSwizzle sw         = CU_TENSOR_MAP_SWIZZLE_NONE;
  int                mask       = 0;
  if (innerBytes > 64) {
    sw   = CU_TENSOR_MAP_SWIZZLE_128B;
    mask = 7;
  } else if (innerBytes > 32) {
    sw   = CU_TENSOR_MAP_SWIZZLE_64B;
    mask = 3;
  } else if (innerBytes > 16) {
    sw   = CU_TENSOR_MAP_SWIZZLE_32B;
    mask = 1;
  }
  cuuint64_t dims[2]    = {cols, rows};
  cuuint64_t strides[1] = {cols * elemBytes};
  cuuint32_t box[2]     = {boxCols, boxRows};
  cuuint32_t estr[2]    = {1, 1};
  CUresult   r = encodeTiled()(tm, dt, 2, const_cast<void*>(base), dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                               sw, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) fail(B200MOL_ERR_CUDA, "cuTensorMapEncodeTiled failed (%d)", static_cast<int>(r));
  return mask;
}

// ---- device ----
__device__ __forceinline__ uint32_t smemAddr(const void* p) { return static_cast<uint32_t>(__cvta_generic_to_shared(p)); }

__device__ __forceinline__ void mbarInit(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smemAddr(bar)), "r"(count));
}
__device__ __forceinline__ void fenceBarrierInit() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
__device__ __forceinline__ void fenceProxyAsync() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }

__device__ __forceinline__ void mbarExpectTx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smemAddr(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbarArrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smemAddr(bar)) : "memory");
}
__device__ __forceinline__ bool mbarTryWait(uint64_t* bar, uint32_t parity) {
  uint32_t ok;
  asm volatile(
    "{\n\t.reg .pred p;\n\t"
    "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
    "selp.u32 %0, 1, 0, p;\n\t}"
    : "=r"(ok)
    : "r"(smemAddr(bar)), "r"(parity)
    : "memory");
  return ok != 0;
}
__device__ __forceinline__ void mbarWait(uint64_t* bar, uint32_t parity) {
  while (!mbarTryWait(bar, parity)) {
  }
}

// 2-D tiled TMA load: coordinates (c0 = innermost element index, c1 = row index).
__device__ __forceinline__ void tmaLoad2D(void* smemDst, const CUtensorMap* tm, int c0, int c1, uint64_t* bar) {
  asm volatile(
    "cp.async.bulk.tensor.2d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];" ::"r"(
      smemAddr(smemDst)),
    "l"(reinterpret_cast<uint64_t>(tm)), "r"(smemAddr(bar)), "r"(c0), "r"(c1)
    : "memory");
}
// The same load delivered to every CTA of the cluster named in ctaMask, at the same shared-memory offsets (data and
// mbarrier) in each of them.
__device__ __forceinline__ void tmaLoad2DMulticast(void* smemDst, const CUtensorMap* tm, int c0, int c1, uint64_t* bar,
                                                   uint16_t ctaMask) {
  asm volatile(
    "cp.async.bulk.tensor.2d.shared::cluster.global.tile.mbarrier::complete_tx::bytes.multicast::cluster [%0], [%1, {%3, %4}], "
    "[%2], %5;" ::"r"(smemAddr(smemDst)),
    "l"(reinterpret_cast<uint64_t>(tm)), "r"(smemAddr(bar)), "r"(c0), "r"(c1), "h"(ctaMask)
    : "memory");
}
// 1-D bulk copy global -> shared memory (16-byte aligned addresses, size a multiple of 16), completing on `bar`.
__device__ __forceinline__ void bulkLoad1D(void* smemDst, const void* src, uint32_t bytes, uint64_t* bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(smemAddr(smemDst)),
               "l"(reinterpret_cast<uint64_t>(src)), "r"(bytes), "r"(smemAddr(bar))
               : "memory");
}
// arrive on the barrier at the same offset in CTA `rank` of the cluster
__device__ __forceinline__ void mbarArriveRemote(uint64_t* bar, uint32_t rank) {
  asm volatile(
    "{\n\t.reg .b32 r;\n\tmapa.shared::cluster.u32 r, %0, %1;\n\tmbarrier.arrive.shared::cluster.b64 _, [r];\n\t}" ::"r"(
      smemAddr(bar)),
    "r"(rank)
    : "memory");
}
__device__ __forceinline__ uint32_t clusterCtaRank() {
  uint32_t r;
  asm volatile("mov.u32 %0, %%cluster_ctarank;" : "=r"(r));
  return r;
}
__device__ __forceinline__ void clusterSync() {
  asm volatile("barrier.cluster.arrive.release.aligned;\n\tbarrier.cluster.wait.acquire.aligned;" ::: "memory");
}
__device__ __forceinline__ void tmaPrefetchDesc(const CUtensorMap* tm) {
  asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(tm)) : "memory");
}

}  // namespace b200
