// async_copy.cuh -- Hopper's asynchronous copy path, written once for the kernels that use it: the ring GEMV
// (gemv_ring_impl.cuh), the integer tensor-core GEMM (gemm_imma.cu), the wgmma GEMM (gemm_tc.cu) and the decode attention
// (attention.cu).  TMA bulk copies land in shared memory and complete on an mbarrier; consumers wait on the barrier by phase
// parity.  Every mbarrier and bulk-copy instruction of those kernels is here, with the shared loads two of them share, and
// the host side: the 2-D tensor maps the TMA tile loads read.
// Addresses of shared memory are 32-bit shared-window addresses (smem_u32), as the instructions take them.
#pragma once
#include <cuda.h>

#include "nsb.cuh"

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

// ---- mbarriers -----------------------------------------------------------------------------------------------------------
__device__ __forceinline__ void mbar_init(uint32_t bar, int count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count) : "memory");
}
// after the inits, before any other thread or the TMA unit uses the barriers (a __syncthreads must still follow)
__device__ __forceinline__ void fence_mbar_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
// one arrival that also announces `bytes` of copies completing on this phase
__device__ __forceinline__ void mbar_expect_tx(uint32_t bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint32_t bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(bar) : "memory");
}
// Spins until the phase of parity `parity` has completed.  The barrier only knows its current phase: a wait issued a whole
// phase early returns at once, as if that phase were the one before it.  So a waiter must never run ahead of the barrier --
// each barrier is waited on by waiters that observe every one of its phases in order.
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity) {
  uint32_t ok;
  do {
    asm volatile(
        "{\n"
        ".reg .pred p;\n"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n"
        "selp.u32 %0, 1, 0, p;\n"
        "}\n"
        : "=r"(ok)
        : "r"(bar), "r"(parity)
        : "memory");
  } while (!ok);
}

// ---- TMA: global -> shared, completion on an mbarrier ------------------------------------------------------------------------
// 1-D bulk copy (SASS: UBLKCP)
__device__ __forceinline__ void bulk_g2s(uint32_t dst, const void* src, uint32_t bytes, uint32_t bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(dst), "l"(src),
               "r"(bytes), "r"(bar)
               : "memory");
}
// 2-D tile of a tensor map at element (x, y) (SASS: UTMALDG)
__device__ __forceinline__ void tma_2d(uint32_t dst, const CUtensorMap* map, int x, int y, uint32_t bar) {
  asm volatile("cp.async.bulk.tensor.2d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3}], [%4];" ::"r"(dst),
               "l"(map), "r"(x), "r"(y), "r"(bar)
               : "memory");
}
__device__ __forceinline__ void prefetch_tensormap(const CUtensorMap* map) {
  asm volatile("prefetch.tensormap [%0];" ::"l"(map) : "memory");
}

// ---- TMA: shared -> global ---------------------------------------------------------------------------------------------------
// makes this thread's generic-proxy shared-memory writes visible to the async proxy (bulk copies, wgmma operands)
__device__ __forceinline__ void fence_proxy_async() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }
// 1-D bulk store into this thread's open bulk group; bulk_commit closes the group, bulk_wait_all waits until every committed
// group has completed (shared memory may not be reused or released before that)
__device__ __forceinline__ void bulk_s2g(void* dst, uint32_t src, uint32_t bytes) {
  asm volatile("cp.async.bulk.global.shared::cta.bulk_group [%0], [%1], %2;" ::"l"(dst), "r"(src), "r"(bytes) : "memory");
}
__device__ __forceinline__ void bulk_commit() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
__device__ __forceinline__ void bulk_wait_all() { asm volatile("cp.async.bulk.wait_group 0;" ::: "memory"); }

// ---- shared loads --------------------------------------------------------------------------------------------------------
__device__ __forceinline__ uint2 lds64(uint32_t a) {
  uint2 r;
  asm volatile("ld.shared.v2.u32 {%0,%1}, [%2];" : "=r"(r.x), "=r"(r.y) : "r"(a));
  return r;
}
__device__ __forceinline__ uint4 lds128(uint32_t a) {
  uint4 r;
  asm volatile("ld.shared.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w) : "r"(a));
  return r;
}

// ---- host: tensor maps ---------------------------------------------------------------------------------------------------
using EncodeTiledFn = decltype(&cuTensorMapEncodeTiled);
// cuTensorMapEncodeTiled from the driver, looked up once.  Null, with the error set, when the driver does not export it.
inline EncodeTiledFn ns_tensor_map_encoder() {
  static EncodeTiledFn fn = nullptr;
  if (!fn) {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult qres;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &qres) == cudaSuccess &&
        qres == cudaDriverEntryPointSuccess)
      fn = (EncodeTiledFn)p;
    else
      ns_set_error("cuTensorMapEncodeTiled not available from the driver");
  }
  return fn;
}
// A 2-D map over `rows` rows of `cols` elements, `pitch` bytes apart, read in boxes of box_cols x box_rows elements: element
// strides 1, no interleave, 128-byte L2 promotion, no out-of-bounds fill.  `what` names the tensor in the error text.
inline int ns_tensor_map_2d(CUtensorMap* map, CUtensorMapDataType type, const void* base, uint64_t cols, uint64_t rows,
                            uint64_t pitch, uint32_t box_cols, uint32_t box_rows, CUtensorMapSwizzle swizzle, const char* what) {
  const EncodeTiledFn enc = ns_tensor_map_encoder();
  if (!enc) return NS_E_CUDA;
  const cuuint64_t dims[2] = {cols, rows}, strides[1] = {pitch};
  const cuuint32_t box[2] = {box_cols, box_rows}, es[2] = {1, 1};
  const CUresult r = enc(map, type, 2, (void*)base, dims, strides, box, es, CU_TENSOR_MAP_INTERLEAVE_NONE, swizzle,
                         CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r == CUDA_SUCCESS) return NS_OK;
  ns_set_error("cuTensorMapEncodeTiled(%s) failed: %d", what, (int)r);
  return NS_E_CUDA;
}
