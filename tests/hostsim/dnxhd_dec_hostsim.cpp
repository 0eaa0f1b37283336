// tests/hostsim/dnxhd_dec_hostsim.cpp -- TEST INFRASTRUCTURE, NOT PRODUCT.
// The product's DNxHD decoder (libav_b200/csrc/dnxhd_dec.cu with dnxhd_dec.cuh: both stage kernels, the probe, the checks and the entry
// points) compiled UNCHANGED as host C++.  Its threads run one after the other; the entropy stage is launched with one thread per CTA here
// (DD_ENTROPY_THREADS), for which its table staging needs no barrier, so the suite runs the product's own row decoder.
#include "shim/cuda_runtime.h"
#include "../../libav_b200/csrc/dnxhd_dec.cu"
