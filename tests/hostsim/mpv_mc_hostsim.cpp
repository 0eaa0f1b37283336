// tests/hostsim/mpv_mc_hostsim.cpp -- TEST INFRASTRUCTURE, NOT PRODUCT.
// The product's mpegvideo motion compensation (libav_b200/csrc/mpv_mc.cu + mpv_mc_block.cuh: the picture checks, the launch and the
// per-lane kernel body; with mpv_obmc.cuh and h263_lf.cuh, OBMC pictures and the H.263 loop filter) compiled UNCHANGED as host C++: a
// launch runs the kernel body once per thread, one after the other, which is exact because the lanes of a macroblock never communicate.
// Of the residual stages of the flush point only the Xvid IDCT is in the host build (xvid_idct_hostsim.cpp); the others report an error.
#include "shim/cuda_runtime.h"
#include "../../libav_b200/csrc/mpv_mc.cu"
