// tests/hostsim/prores_hostsim.cpp -- TEST INFRASTRUCTURE, NOT PRODUCT.
// The product's ProRes reconstruction (libav_b200/csrc/prores.cu: the thread-per-block kernels, the picture addressing, both entry points,
// the table slot and ff_proresdsp_init_cuda) compiled UNCHANGED as host C++.  Every call takes the thread-per-block kernels here: the staged
// kernel needs warps and shared memory and is checked on the GPU only.
#include "shim/cuda_runtime.h"
#include "../../libav_b200/csrc/prores.cu"
