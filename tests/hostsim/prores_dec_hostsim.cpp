// tests/hostsim/prores_dec_hostsim.cpp -- TEST INFRASTRUCTURE, NOT PRODUCT.
// The product's ProRes decoder (libav_b200/csrc/prores_dec.cu with prores_dec.cuh: the offset, entropy and alpha kernels, the probe, the
// checks and the entry points) compiled UNCHANGED as host C++.  Its threads run one after the other, the entropy stage with one thread per
// CTA (PRD_THREADS); the put stage is prores.cu's thread-per-block picture kernel, from prores_hostsim.cpp in the same library.
#include "shim/cuda_runtime.h"
#include "../../libav_b200/csrc/prores_dec.cu"

// the decoder's tables, in the order of ref_prores_dec_tables (oracle/refbuild/refapi_prores_dec.c): both scans, the DC and AC codebooks,
// run_to_cb_index, lev_to_cb_index, FIRST_DC_CB.  Returns the count.
extern "C" int hostsim_prores_dec_tables(int32_t *out)
{
    using namespace avb;
    int n = 0;
    for (int s = 0; s < 2; s++) for (int i = 0; i < 64; i++) out[n++] = pe_scan[s][i];
    for (int i = 0; i < 4; i++) out[n++] = pe_dc_codebook[i];
    for (int i = 0; i < 7; i++) out[n++] = pe_ac_codebook[i];
    for (int i = 0; i < 16; i++) out[n++] = pe_run_to_cb[i];
    for (int i = 0; i < 10; i++) out[n++] = pe_lev_to_cb[i];
    out[n++] = PE_FIRST_DC_CB;
    return n;
}
