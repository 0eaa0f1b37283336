// tests/hostsim/faan_idct_hostsim.cpp -- TEST INFRASTRUCTURE, NOT PRODUCT.
// The product's FAAN transforms (libav_b200/csrc/faan_idct.cu: the thread-per-block IDCT kernel, ff_faanidct_batch_cuda, the table slots,
// and the ff_faandct / ff_faandct248 kernel behind ff_fdct_batch_cuda 6 / 7) compiled UNCHANGED as host C++, where plain float and double
// operators round like the reference's x86-64 build.  Every IDCT batch takes the thread-per-block kernel here: the staged kernel
// (idctdsp.cu) needs warps and shared memory and is checked on the GPU only, like the fused inverse quantisers in front of it.
#include "shim/cuda_runtime.h"
#include "../../libav_b200/csrc/faan_idct.cu"

extern "C" {
// ff_fdct_batch_cuda(6 | 7, ...) is a GPU-only entry point (me_cmp.cu); this reaches the same launcher
int hostsim_faan_fdct(int which, int16_t *blocks, size_t n) { return avb::faan_fdct_launch(which, blocks, n, nullptr); }
// the flush's transform 3 with a fused inverse quantiser (capi_idct.cu, not in the host build)
int ff_mpeg_dequant_faanidct_batch_cuda(int, const FFMpegDequantTables *, const FFMpegDequantBlock *, int16_t *, uint8_t *, const uint32_t *,
                                        ptrdiff_t, size_t, int, int, void *)
{
    avb::set_error_msg("ff_mpeg_dequant_faanidct_batch_cuda", "not in the host build");
    return -1;
}
}
