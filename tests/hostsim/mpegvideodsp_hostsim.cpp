// tests/hostsim/mpegvideodsp_hostsim.cpp -- TEST INFRASTRUCTURE, NOT PRODUCT.
// The MpegVideoDSPContext slots (libav_b200/csrc/mpegvideodsp.cu: staging, the slot kernel with the GMC arithmetic of mpv_gmc.cuh, the
// ff_mpegvideodsp_init_cuda hook) compiled UNCHANGED as host C++.  "Device" memory is host memory here and the scratch pool is poisoned,
// so a slot that reads a sample it did not stage gives a different block.  S-VOPs in the batched MC come with mpv_mc.cu (mpv_mc_hostsim.cpp).
#include "shim/cuda_runtime.h"
#include "../../libav_b200/csrc/mpegvideodsp.cu"
