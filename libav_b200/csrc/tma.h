// libav_b200/csrc/tma.h -- tensor-map encoding and the mbarrier / bulk-tensor PTX the TMA-fed kernels share.
// cuTensorMapEncodeTiled is looked up through the runtime's driver entry point: the library does not link libcuda.
#pragma once
#include "common.cuh"
#include <cuda.h>

namespace avb {

// rank-`rank` tiled tensor map without swizzle or interleave; dims / box in elements (innermost first), strides in bytes for dims 1..rank-1
inline bool tma_encode(CUtensorMap *tm, CUtensorMapDataType type, int rank, const void *base, const cuuint64_t *dims,
                       const cuuint64_t *strides, const cuuint32_t *box, CUtensorMapSwizzle swz = CU_TENSOR_MAP_SWIZZLE_NONE)
{
    typedef CUresult (*EncodeFn)(CUtensorMap *, CUtensorMapDataType, cuuint32_t, void *, const cuuint64_t *, const cuuint64_t *,
                                 const cuuint32_t *, const cuuint32_t *, CUtensorMapInterleave, CUtensorMapSwizzle,
                                 CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
    static EncodeFn fn = nullptr;
    static bool tried = false;
    if (!tried) {
        tried = true;
        void *p = nullptr;
        cudaDriverEntryPointQueryResult q;
        if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) == cudaSuccess && q == cudaDriverEntryPointSuccess) fn = (EncodeFn)p;
        else cudaGetLastError();
    }
    if (!fn) return false;
    const cuuint32_t estr[5] = { 1, 1, 1, 1, 1 };
    return fn(tm, type, (cuuint32_t)rank, const_cast<void *>(base), dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE, swz,
              CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) == CUDA_SUCCESS;
}

#ifdef __CUDACC__
__device__ __forceinline__ void mbar_init(unsigned mbar_s, int count)
{ asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" :: "r"(mbar_s), "r"(count) : "memory"); }
__device__ __forceinline__ void mbar_init_fence() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
__device__ __forceinline__ void mbar_expect_tx(unsigned mbar_s, int bytes)
{ asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" :: "r"(mbar_s), "r"(bytes) : "memory"); }
__device__ __forceinline__ void mbar_wait(unsigned mbar_s, unsigned parity)
{
    asm volatile("{\n.reg .pred p;\nAVB_MBAR_WAIT_%=:\nmbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n@p bra AVB_MBAR_DONE_%=;\nbra AVB_MBAR_WAIT_%=;\nAVB_MBAR_DONE_%=:\n}"
                 :: "r"(mbar_s), "r"(parity) : "memory");
}
// generic-proxy accesses to a buffer before the async proxy (TMA) reuses it
__device__ __forceinline__ void fence_proxy_async() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }
__device__ __forceinline__ void tma_load_3d(unsigned dst_s, const CUtensorMap *tm, int x, int y, int z, unsigned mbar_s)
{
    asm volatile("cp.async.bulk.tensor.3d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3, %4}], [%5];"
                 :: "r"(dst_s), "l"(reinterpret_cast<uint64_t>(tm)), "r"(x), "r"(y), "r"(z), "r"(mbar_s) : "memory");
}
__device__ __forceinline__ void tma_load_2d(unsigned dst_s, const CUtensorMap *tm, int x, int y, unsigned mbar_s)
{
    asm volatile("cp.async.bulk.tensor.2d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3}], [%4];"
                 :: "r"(dst_s), "l"(reinterpret_cast<uint64_t>(tm)), "r"(x), "r"(y), "r"(mbar_s) : "memory");
}
// an L2 cache policy (createpolicy) for the global-memory side of the two operations below
__device__ __forceinline__ uint64_t l2_policy_evict_first()
{ uint64_t p; asm volatile("createpolicy.fractional.L2::evict_first.b64 %0, 1.0;" : "=l"(p)); return p; }
// tma_load_3d with the policy attached
__device__ __forceinline__ void tma_load_3d_hint(unsigned dst_s, const CUtensorMap *tm, int x, int y, int z, unsigned mbar_s, uint64_t policy)
{
    asm volatile("cp.async.bulk.tensor.3d.shared::cluster.global.tile.mbarrier::complete_tx::bytes.L2::cache_hint [%0], [%1, {%2, %3, %4}], [%5], %6;"
                 :: "r"(dst_s), "l"(reinterpret_cast<uint64_t>(tm)), "r"(x), "r"(y), "r"(z), "r"(mbar_s), "l"(policy) : "memory");
}
// shared -> global bulk tensor store (bulk async-group completion) with the policy attached; the source must have been made visible
// with fence_proxy_async()
__device__ __forceinline__ void tma_store_3d_hint(const CUtensorMap *tm, int x, int y, int z, unsigned src_s, uint64_t policy)
{
    asm volatile("cp.async.bulk.tensor.3d.global.shared::cta.tile.bulk_group.L2::cache_hint [%0, {%1, %2, %3}], [%4], %5;"
                 :: "l"(reinterpret_cast<uint64_t>(tm)), "r"(x), "r"(y), "r"(z), "r"(src_s), "l"(policy) : "memory");
}
__device__ __forceinline__ void bulk_commit() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
template <int N> __device__ __forceinline__ void bulk_wait_read() { asm volatile("cp.async.bulk.wait_group.read %0;" :: "n"(N) : "memory"); }
template <int N> __device__ __forceinline__ void bulk_wait() { asm volatile("cp.async.bulk.wait_group %0;" :: "n"(N) : "memory"); }
__device__ __forceinline__ void sts128(unsigned a, uint4 v)
{ asm volatile("st.shared.v4.u32 [%0], {%1,%2,%3,%4};" :: "r"(a), "r"(v.x), "r"(v.y), "r"(v.z), "r"(v.w) : "memory"); }
__device__ __forceinline__ uint4 lds128(unsigned a)
{ uint4 r; asm volatile("ld.shared.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w) : "r"(a) : "memory"); return r; }
__device__ __forceinline__ uint2 lds64(unsigned a)
{ uint2 r; asm volatile("ld.shared.v2.u32 {%0,%1}, [%2];" : "=r"(r.x), "=r"(r.y) : "r"(a) : "memory"); return r; }
// read-only tables in shared memory (written once before a barrier): not volatile, the compiler may schedule them freely
__device__ __forceinline__ uint2 lds64_ro(unsigned a)
{ uint2 r; asm("ld.shared.v2.u32 {%0,%1}, [%2];" : "=r"(r.x), "=r"(r.y) : "r"(a)); return r; }
#endif

}  // namespace avb
