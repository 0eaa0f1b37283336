// tests/hostsim/xvid_idct_hostsim.cpp -- TEST INFRASTRUCTURE, NOT PRODUCT.
// The product's Xvid IDCT (libav_b200/csrc/xvid_idct.cu: the thread-per-block kernel, the batched entry point, the table slots and
// ff_xvid_idct_init_cuda) compiled UNCHANGED as host C++.  Every batch takes the thread-per-block kernel here: the staged kernel it shares
// with the simple IDCT (idctdsp.cu) needs warps and shared memory and is checked on the GPU only.
#include "shim/cuda_runtime.h"
#include "../../libav_b200/csrc/xvid_idct.cu"
