// tests/hostsim/mpv_mc_hostsim.cpp -- TEST INFRASTRUCTURE, NOT PRODUCT.
// The product's mpegvideo motion compensation (libav_b200/csrc/mpv_mc.cu + mpv_mc_block.cuh: the picture checks, the launch and the
// per-lane kernel body) compiled UNCHANGED as host C++: a launch runs the kernel body once per thread, one after the other, which is
// exact because the lanes of a macroblock never communicate.  The residual stages of the flush point live in other files and are not
// part of this build: here they only report an error.
#include "shim/cuda_runtime.h"
#include <string>
#define __grid_constant__
static inline unsigned atomicAdd(unsigned *p, unsigned v) { const unsigned o = *p; *p = o + v; return o; }
uint3 threadIdx, blockIdx;
dim3 blockDim, gridDim;
#include "../../libav_b200/csrc/mpv_mc.cu"

namespace avb {
static std::string g_err;
void set_error_msg(const char *where, const char *msg) { if (g_err.empty()) g_err = std::string(where) + ": " + msg; }
void set_error(const char *where, cudaError_t) { set_error_msg(where, "hostsim error"); }
int check_launch(const char *) { return 0; }
void enter() {}
}

#define NOT_HERE(name, ...) extern "C" int name(__VA_ARGS__) { avb::set_error_msg(#name, "not in the host build"); return -1; }
NOT_HERE(ff_simple_idct_batch_cuda, int, int16_t *, uint8_t *, const uint32_t *, ptrdiff_t, size_t, int, int, void *)
NOT_HERE(ff_xvid_idct_batch_cuda, int, int16_t *, uint8_t *, const uint32_t *, ptrdiff_t, size_t, int, int, void *)
NOT_HERE(ff_mpeg_dequant_idct_batch_cuda, int, const FFMpegDequantTables *, const FFMpegDequantBlock *, int16_t *, uint8_t *, const uint32_t *,
         ptrdiff_t, size_t, int, int, void *)
NOT_HERE(ff_mpeg_dequant_xvid_idct_batch_cuda, int, const FFMpegDequantTables *, const FFMpegDequantBlock *, int16_t *, uint8_t *, const uint32_t *,
         ptrdiff_t, size_t, int, int, void *)

extern "C" const char *hostsim_last_error() { return avb::g_err.c_str(); }
extern "C" void hostsim_clear_error() { avb::g_err.clear(); }
