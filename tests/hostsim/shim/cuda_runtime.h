/* tests/hostsim/shim/cuda_runtime.h -- TEST INFRASTRUCTURE, NOT PRODUCT.
 *
 * Just enough of the CUDA runtime's surface, implemented on the host, for tests/hostsim/ to compile the product's
 * thread-independent slot path (libav_b200/csrc/slots.cu + h264dsp.cuh) as plain C++ with g++: "device memory" is host
 * memory, copies are memcpy, a launch runs the kernel body once per (block, thread) index in sequence.  That is only
 * valid for kernels whose threads do not communicate (no shared memory, shuffles, barriers or atomics) -- exactly the
 * per-call slot kernel; every other kernel of the product is checked on the GPU only.
 */
#ifndef HOSTSIM_CUDA_RUNTIME_H
#define HOSTSIM_CUDA_RUNTIME_H
#include <stdint.h>
#include <stddef.h>
#include <stdlib.h>
#include <string.h>

#define __device__
#define __host__
#define __global__
#define __forceinline__ inline
#define __launch_bounds__(...)
#define __shared__
#define __grid_constant__
#define __align__(n) __attribute__((aligned(n)))

typedef int cudaError_t;
enum { cudaSuccess = 0 };
typedef struct hostsim_stream *cudaStream_t;
typedef struct hostsim_event *cudaEvent_t;
enum cudaMemcpyKind { cudaMemcpyHostToHost, cudaMemcpyHostToDevice, cudaMemcpyDeviceToHost, cudaMemcpyDeviceToDevice };

struct uint3 { unsigned x, y, z; };
struct int2 { int x, y; };
struct int4 { int x, y, z, w; };
struct uint2 { unsigned x, y; };
struct uint4 { unsigned x, y, z, w; };
struct dim3 {
    unsigned x, y, z;
    dim3(unsigned x_ = 1, unsigned y_ = 1, unsigned z_ = 1) : x(x_), y(y_), z(z_) {}
};
extern uint3 threadIdx, blockIdx;
extern dim3 blockDim, gridDim;

static inline cudaError_t cudaMemcpyAsync(void *d, const void *s, size_t n, cudaMemcpyKind, cudaStream_t) { memcpy(d, s, n); return cudaSuccess; }
static inline cudaError_t cudaStreamSynchronize(cudaStream_t) { return cudaSuccess; }
enum { cudaStreamNonBlocking = 1 };
static inline cudaError_t cudaStreamCreateWithFlags(cudaStream_t *s, unsigned) { *s = nullptr; return cudaSuccess; }
static inline cudaError_t cudaStreamDestroy(cudaStream_t) { return cudaSuccess; }
static inline cudaError_t cudaGetLastError() { return cudaSuccess; }
static inline const char *cudaGetErrorString(cudaError_t) { return "hostsim"; }

static inline uint2 make_uint2(unsigned x, unsigned y) { uint2 r = { x, y }; return r; }
static inline uint4 make_uint4(unsigned x, unsigned y, unsigned z, unsigned w) { uint4 r = { x, y, z, w }; return r; }
static inline int2 make_int2(int x, int y) { int2 r = { x, y }; return r; }
template <class T> static inline T __ldg(const T *p) { return *p; }
static inline int __vimin_s32_relu(int a, int b) { const int m = a < b ? a : b; return m < 0 ? 0 : m; }
static inline unsigned __vimin_s16x2_relu(unsigned a, unsigned b)
{
    unsigned r = 0;
    for (int k = 0; k < 2; k++) {
        const int x = (int16_t)(a >> (16 * k)), y = (int16_t)(b >> (16 * k));
        int m = x < y ? x : y;
        if (m < 0) m = 0;
        r |= (unsigned)(m & 0xffff) << (16 * k);
    }
    return r;
}
/* kernels that synchronise their threads (shared-memory tiles) cannot run one thread after the other: they must never be launched here */
static inline void __syncthreads() { abort(); }

static inline cudaError_t cudaMalloc(void **p, size_t n) { *p = malloc(n ? n : 1); if (*p) memset(*p, 0xA7, n); return *p ? cudaSuccess : 2; }
template <class T> static inline cudaError_t cudaMalloc(T **p, size_t n) { return cudaMalloc((void **)p, n); }
static inline cudaError_t cudaFree(void *p) { free(p); return cudaSuccess; }
static inline cudaError_t cudaMemcpy(void *d, const void *s, size_t n, cudaMemcpyKind) { memcpy(d, s, n); return cudaSuccess; }
static inline cudaError_t cudaMemcpy2DAsync(void *d, size_t dp, const void *s, size_t sp, size_t w, size_t h, cudaMemcpyKind, cudaStream_t)
{
    for (size_t y = 0; y < h; y++) memcpy((char *)d + y * dp, (const char *)s + y * sp, w);
    return cudaSuccess;
}
static inline cudaError_t cudaMemsetAsync(void *d, int v, size_t n, cudaStream_t) { memset(d, v, n); return cudaSuccess; }
static inline cudaError_t cudaMemset2DAsync(void *d, size_t dp, int v, size_t w, size_t h, cudaStream_t)
{
    for (size_t y = 0; y < h; y++) memset((char *)d + y * dp, v, w);
    return cudaSuccess;
}
enum cudaFuncAttribute { cudaFuncAttributeMaxDynamicSharedMemorySize = 8 };
template <class F> static inline cudaError_t cudaFuncSetAttribute(F, cudaFuncAttribute, int) { return cudaSuccess; }

static inline int min(int a, int b) { return a < b ? a : b; }
static inline int max(int a, int b) { return a > b ? a : b; }
static inline unsigned min(unsigned a, unsigned b) { return a < b ? a : b; }
static inline unsigned max(unsigned a, unsigned b) { return a > b ? a : b; }
static inline unsigned __byte_perm(unsigned a, unsigned b, unsigned sel)
{
    const uint64_t v = ((uint64_t)b << 32) | a;
    unsigned r = 0;
    for (int i = 0; i < 4; i++) {
        const unsigned s = (sel >> (4 * i)) & 0xf;
        unsigned byte = (unsigned)(v >> (8 * (s & 7))) & 0xff;
        if (s & 8) byte = (byte & 0x80) ? 0xff : 0;
        r |= byte << (8 * i);
    }
    return r;
}
static inline int atomicMin(int *p, int v) { const int old = *p; if (v < old) *p = v; return old; }      /* threads run one after the other here */
static inline unsigned atomicAdd(unsigned *p, unsigned v) { const unsigned old = *p; *p = old + v; return old; }
static inline int __mulhi(int a, int b) { return (int)(((int64_t)a * b) >> 32); }
static inline size_t __cvta_generic_to_shared(const void *p) { return (size_t)p; }

namespace hostsim {
/* a launch = the kernel body once per (block, thread) index, one after the other; the kernel is named inside a generic lambda so that
 * default arguments and template specialisations work exactly as in a direct call */
template <class F> struct Launch {
    F call;
    dim3 grid, block;
    template <class... A> void operator()(A... args) const
    {
        gridDim = grid; blockDim = block;
        for (unsigned bz = 0; bz < grid.z; bz++) for (unsigned by = 0; by < grid.y; by++) for (unsigned bx = 0; bx < grid.x; bx++)
            for (unsigned tz = 0; tz < block.z; tz++) for (unsigned ty = 0; ty < block.y; ty++) for (unsigned tx = 0; tx < block.x; tx++) {
                blockIdx = { bx, by, bz }; threadIdx = { tx, ty, tz };
                call(args...);
            }
    }
};
template <class F> Launch<F> launch(F f, dim3 g, dim3 b) { return Launch<F>{ f, g, b }; }
}
#define AVB_LAUNCH(kernel, grid, block, smem, stream) hostsim::launch([&](auto... a_) { kernel(a_...); }, grid, block)

#endif
