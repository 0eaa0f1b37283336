// tests/hostsim/mpv_quant_hostsim.cpp -- TEST INFRASTRUCTURE, NOT PRODUCT.
// The product's encoder quantiser (libav_b200/csrc/mpv_quant.cu: the batched entry point, the state objects, the kernel with the plain
// quantiser of mpv_quant.cuh, the trellis, noise reduction, clip and elimination, and the dct_quantize slots) compiled UNCHANGED as host
// C++: a launch runs the kernel body once per thread, one after the other.  That is exact because a thread only ever touches its own
// column of the trellis tables and its own block; the noise-reduction sums, which the device reduces over the warp, are added directly
// (AVB_HOSTSIM).  The VLC table cache it shares with the metrics comes from me_cmp_enc_hostsim.cpp.
#include "shim/cuda_runtime.h"
#include "../../libav_b200/csrc/mpv_quant.cu"
