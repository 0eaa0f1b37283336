// libav_b200/csrc/common.cuh -- shared device/host helpers for the sm_90a DSP kernels.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <stddef.h>
#include <stdio.h>
#include <string.h>

namespace avb {

// ---- sticky error channel (the reference's DSP slots return void; see include/avdsp_b200.h) ----
void set_error(const char *where, cudaError_t e);
void set_error_msg(const char *where, const char *msg);
int  check_launch(const char *where);   // cudaGetLastError() -> sticky error, returns 0/-1

#define AVB_CUDA(call, where)                                              \
    do {                                                                   \
        cudaError_t e__ = (call);                                          \
        if (e__ != cudaSuccess) { avb::set_error(where, e__); return -1; } \
    } while (0)

// Kernel launch.  The product always expands to the <<<>>> form; tests/hostsim/ (test infrastructure, CPU suite) defines this
// macro first and compiles the thread-independent slot kernels as host C++ so that the slot plumbing is checked without a GPU.
#ifndef AVB_LAUNCH
#define AVB_LAUNCH(kernel, grid, block, smem, stream) kernel<<<(grid), (block), (smem), (stream)>>>
#endif

void enter();                   // make the device avb200_init() chose current in the calling thread (first statement of every public entry point)
int sm_count();                 // multiprocessor count of the current device (cached)
int tuning(const char *key);    // test knob set through avb200_set_tuning(); 0 when unset
// the arguments the 8-bit intra wavefront needs (h264intra.cu); false = refused with a message.  mbs: const FFH264IntraMB *
bool h264_intra_args_ok(const char *where, const void *mbs, const int16_t *coeffs, size_t coeff_stride, const uint8_t *nnzc, const uint8_t *luma,
                        const uint8_t *cb, const uint8_t *cr, int linesize, int uvlinesize, const uint32_t *progress);

// ---- device helpers ------------------------------------------------------------------------
#ifdef AVB_HOSTSIM
// tests/hostsim/ (CPU suite) compiles the thread-independent kernels as host C++: the PTX helpers below get their plain definitions there
inline uint4 ldg_stream(const void *p) { return *reinterpret_cast<const uint4 *>(p); }
inline uint2 ldg_stream8(const void *p) { return *reinterpret_cast<const uint2 *>(p); }
inline void stg_stream(void *p, uint4 v) { *reinterpret_cast<uint4 *>(p) = v; }
inline void stg_stream8(void *p, uint2 v) { *reinterpret_cast<uint2 *>(p) = v; }
inline void cp_async16(void *smem, const void *gmem, bool valid) { if (valid) memcpy(smem, gmem, 16); else memset(smem, 0, 16); }
inline void cp_async4(void *smem, const void *gmem) { memcpy(smem, gmem, 4); }
inline void cp_async_commit() {}
template <int N> inline void cp_async_wait() {}
inline uint32_t pack_sat_u8(int b0, int b1, uint32_t hi16)
{
    const uint32_t s0 = (uint32_t)(b0 < 0 ? 0 : b0 > 255 ? 255 : b0), s1 = (uint32_t)(b1 < 0 ? 0 : b1 > 255 ? 255 : b1);
    return (hi16 << 16) | (s1 << 8) | s0;
}
#else
// streaming 128-bit global accesses (data touched exactly once: keep it out of L1)
__device__ __forceinline__ uint4 ldg_stream(const void *p)
{
    uint4 r;
    asm volatile("ld.global.nc.L1::no_allocate.v4.u32 {%0,%1,%2,%3}, [%4];"
                 : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w) : "l"(p));
    return r;
}
__device__ __forceinline__ uint2 ldg_stream8(const void *p)
{
    uint2 r;
    asm volatile("ld.global.nc.L1::no_allocate.v2.u32 {%0,%1}, [%2];" : "=r"(r.x), "=r"(r.y) : "l"(p));
    return r;
}
__device__ __forceinline__ void stg_stream(void *p, uint4 v)
{
    asm volatile("st.global.L1::no_allocate.v4.u32 [%0], {%1,%2,%3,%4};"
                 :: "l"(p), "r"(v.x), "r"(v.y), "r"(v.z), "r"(v.w) : "memory");
}
__device__ __forceinline__ void stg_stream8(void *p, uint2 v)
{
    asm volatile("st.global.L1::no_allocate.v2.u32 [%0], {%1,%2};" :: "l"(p), "r"(v.x), "r"(v.y) : "memory");
}

// cp.async 16 B global -> shared (LDGSTS), zero-fill when !valid
__device__ __forceinline__ void cp_async16(void *smem, const void *gmem, bool valid)
{
    unsigned s = (unsigned)__cvta_generic_to_shared(smem);
    int sz = valid ? 16 : 0;
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" :: "r"(s), "l"(gmem), "r"(sz) : "memory");
}
// 4-byte variant (cp.async.ca): side information whose records are only 4- or 8-byte aligned
__device__ __forceinline__ void cp_async4(void *smem, const void *gmem)
{
    unsigned s = (unsigned)__cvta_generic_to_shared(smem);
    asm volatile("cp.async.ca.shared.global [%0], [%1], 4;" :: "r"(s), "l"(gmem) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N> __device__ __forceinline__ void cp_async_wait() { asm volatile("cp.async.wait_group %0;" :: "n"(N) : "memory"); }

// two s32 -> saturated u8, packed under the low 16 bits of `hi16` shifted up:
//   result = (hi16 << 16) | (sat_u8(b1) << 8) | sat_u8(b0)      (SASS: I2IP.U8.S32.SAT)
__device__ __forceinline__ uint32_t pack_sat_u8(int b0, int b1, uint32_t hi16)
{
    uint32_t d;
    asm("cvt.pack.sat.u8.s32.b32 %0, %1, %2, %3;" : "=r"(d) : "r"(b1), "r"(b0), "r"(hi16));
    return d;
}
#endif
// four s32 -> one little-endian word of saturated bytes {p0,p1,p2,p3}
__device__ __forceinline__ uint32_t pack4_sat_u8(int p0, int p1, int p2, int p3)
{
    return pack_sat_u8(p0, p1, pack_sat_u8(p2, p3, 0));
}
__device__ __forceinline__ int byte_of(uint32_t w, int k) { return (int)__byte_perm(w, 0, 0x4440 + k); }
__device__ __forceinline__ int lo16s(uint32_t w) { return (int)(int16_t)(w & 0xffff); }
__device__ __forceinline__ int hi16s(uint32_t w) { return (int)w >> 16; }
__device__ __forceinline__ uint32_t pack16(int lo, int hi) { return __byte_perm((uint32_t)lo, (uint32_t)hi, 0x5410); }
__device__ __forceinline__ int clip_u8(int v) { return min(max(v, 0), 255); }
// arithmetic shift right by a constant.  MULHI = true issues it as IMAD.HI (x * 2^(32-N) >> 32 == x >> N for signed x) on the
// FMA pipe instead of SHF on the ALU pipe -- these kernels are bound by the 16-lane integer ALU pipe, the FMA pipe has slack.
template <int N, bool MULHI> __device__ __forceinline__ int sra(int x) { return MULHI ? __mulhi(x, 1 << (32 - N)) : (x >> N); }

}  // namespace avb
