// tests/hostsim/h263_hostsim.cpp -- TEST INFRASTRUCTURE, NOT PRODUCT.
// The product's H.263 paths compiled UNCHANGED as host C++ through the motion compensation's host build (mpv_mc.cu, which includes
// mpv_obmc.cuh and h263_lf.cuh): OBMC pictures in ff_mpv_motion_batch_cuda, the loop filter's checks, launch and per-thread tile body, and
// the slot kernel.  A launch runs the kernel body once per thread, one after the other, which is exact because the threads never
// communicate.  "Device" memory is
// host memory here, so the slot kernel runs on the caller's samples in place.
#include "mpv_mc_hostsim.cpp"

// the slot kernel on the caller's samples (qscale 0..31)
extern "C" int hostsim_h263_slot(int vert, uint8_t *src, int stride, int qscale)
{
    AVB_LAUNCH(avb::h263_lf_slot_kernel, 1, 32, 0, nullptr)(src, stride, (int)avb::h263_lf_strength_tab[qscale], vert);
    return 0;
}
