// tests/hostsim/slots_hostsim.cpp -- TEST INFRASTRUCTURE, NOT PRODUCT.
//
// The product's per-call slot path (libav_b200/csrc/slots.cu: staging, argument packing, the slot kernel with the device
// arithmetic of h264dsp.cuh, the ff_*_init_cuda table hooks) compiled UNCHANGED as host C++ against shim/cuda_runtime.h, so
// that the CPU suite can drive the H.264 slots exactly like tests/test_gpu_slots.py drives them on the GPU and compare them
// with the oracle.  This library is never loaded by the product and never measured; it exists because the GPU box is not
// always at hand while the slot code changes.  Slots that route through the batched kernels (FDCT, me_cmp, hpel, MPEG-4 qpel,
// pixblock, weight) need warps and shared memory and are not simulated: their launchers fail loudly (runtime_hostsim.cpp).
#include "shim/cuda_runtime.h"
#include "../../libav_b200/csrc/slots.cu"
#include "../../libav_b200/csrc/fdct10.cu"
