// tests/hostsim/runtime_hostsim.cpp -- TEST INFRASTRUCTURE, NOT PRODUCT.
//
// The one runtime of tests/hostsim/libhostsim.so, shared by every unit in it: the launch indices AVB_LAUNCH sets, the product's sticky
// error channel (the first message sticks until avb200_clear_error, as in the GPU build), the device hooks of common.cuh, the scratch
// pool of scratch.h, and the entry points the host build cannot run.  Those are the batched kernels that need warps or shared memory,
// and the residual stages of the mpegvideo flush point whose files are not compiled here: they report an error and return -1.
#include "shim/cuda_runtime.h"
#include <mutex>
#include <string>
#include "common.cuh"
#include "scratch.h"
#include "../../include/avdsp_b200.h"

uint3 threadIdx, blockIdx;
dim3 blockDim, gridDim;

namespace avb {
static std::string g_err;
void set_error_msg(const char *where, const char *msg) { if (g_err.empty()) g_err = std::string(where) + ": " + msg; }
void set_error(const char *where, cudaError_t) { set_error_msg(where, "hostsim error"); }
int check_launch(const char *) { return 0; }
void enter() {}
int sm_count() { return 148; }
// the general scaler is forced onto its two-pass path here: the tile kernels synchronise their threads (swscale_hostsim.cpp)
int tuning(const char *key) { return !strcmp(key, "sws_general_variant") ? 1 : 0; }

static Scratch g_scratch;
static std::recursive_mutex g_mu;
Scratch &scratch() { return g_scratch; }
std::recursive_mutex &scratch_mutex() { return g_mu; }
// real device / pinned allocations come back uninitialised: poison them so that a kernel reading bytes nobody staged cannot pass by luck
static void *grow(void *&p, size_t &n, size_t bytes) { if (n < bytes) { free(p); p = malloc(bytes); memset(p, 0xA7, bytes); n = bytes; } return p; }
void *Scratch::dev(int slot, size_t bytes) { void *p = grow(d_[slot], dn_[slot], bytes); memset(p, 0xA7, bytes); return p; }      // (every call: contents are undefined)
void *Scratch::pinned(size_t bytes) { return grow(h_, hn_, bytes); }
void *Scratch::pinned2(size_t bytes) { void *p = grow(h2_, h2n_, bytes); memset(p, 0x5B, bytes); return p; }
cudaStream_t *Scratch::streams() { return st_; }

int fdct10_launch(int which, int16_t *blocks, size_t n, cudaStream_t st);      // fdct10.cu (slots_hostsim.cpp)
}  // namespace avb

extern "C" {
const char *avb200_last_error(void) { return avb::g_err.c_str(); }
void avb200_clear_error(void) { avb::g_err.clear(); }

#define NOT_SIMULATED(name) { avb::set_error_msg(name, "batched kernel: not simulated on the host"); return -1; }
int ff_me_cmp_batch_cuda(int, int, int, const uint8_t *, const uint8_t *, ptrdiff_t, int, const FFMECmpRecord *, size_t, int32_t *, void *) NOT_SIMULATED("ff_me_cmp_batch_cuda")
int ff_hpel_batch_cuda(const FFHpelRecord *, size_t, uint8_t *, const uint8_t *, ptrdiff_t, void *) NOT_SIMULATED("ff_hpel_batch_cuda")
// the 8-bit transforms are warp kernels (me_cmp.cu, not simulated); the 10-bit ones are thread-per-block (fdct10.cu)
int ff_fdct_batch_cuda(int which, int16_t *blocks, size_t n, void *stream)
{
    if (which == 4 || which == 5) return avb::fdct10_launch(which, blocks, n, (cudaStream_t)stream);
    NOT_SIMULATED("ff_fdct_batch_cuda")
}
int ff_mpeg4_qpel_batch_cuda(const FFQpelRecord *, size_t, uint8_t *, const uint8_t *, ptrdiff_t, void *) NOT_SIMULATED("ff_mpeg4_qpel_batch_cuda")
int ff_pixblock_fdct_batch_cuda(int, const uint8_t *, const uint8_t *, const uint32_t *, const uint32_t *, ptrdiff_t, int16_t *, size_t, void *) NOT_SIMULATED("ff_pixblock_fdct_batch_cuda")
int ff_h264_weight_batch_cuda(const FFH264WeightRecord *, size_t, uint8_t *, const uint8_t *, int, void *) NOT_SIMULATED("ff_h264_weight_batch_cuda")
}

// the residual stages of ff_mpv_flush_pictures_cuda other than the Xvid IDCT (xvid_idct_hostsim.cpp)
#define NOT_HERE(name, ...) extern "C" int name(__VA_ARGS__) { avb::set_error_msg(#name, "not in the host build"); return -1; }
NOT_HERE(ff_simple_idct_batch_cuda, int, int16_t *, uint8_t *, const uint32_t *, ptrdiff_t, size_t, int, int, void *)
NOT_HERE(ff_mpeg_dequant_idct_batch_cuda, int, const FFMpegDequantTables *, const FFMpegDequantBlock *, int16_t *, uint8_t *, const uint32_t *,
         ptrdiff_t, size_t, int, int, void *)
NOT_HERE(ff_mpeg_dequant_xvid_idct_batch_cuda, int, const FFMpegDequantTables *, const FFMpegDequantBlock *, int16_t *, uint8_t *, const uint32_t *,
         ptrdiff_t, size_t, int, int, void *)
