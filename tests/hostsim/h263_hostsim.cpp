// tests/hostsim/h263_hostsim.cpp -- TEST INFRASTRUCTURE, NOT PRODUCT.
// The H263DSPContext slot kernel (libav_b200/csrc/h263_lf.cuh) compiled UNCHANGED as host C++.  "Device" memory is host memory here, so
// the slot kernel runs on the caller's samples in place.  The picture filter and OBMC come with mpv_mc.cu (mpv_mc_hostsim.cpp).
#include "shim/cuda_runtime.h"
#include "../../libav_b200/csrc/h263_lf.cuh"

// the slot kernel on the caller's samples (qscale 0..31)
extern "C" int hostsim_h263_slot(int vert, uint8_t *src, int stride, int qscale)
{
    AVB_LAUNCH(avb::h263_lf_slot_kernel, 1, 32, 0, nullptr)(src, stride, (int)avb::h263_lf_strength_tab[qscale], vert);
    return 0;
}
