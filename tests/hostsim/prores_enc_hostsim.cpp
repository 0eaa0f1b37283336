// tests/hostsim/prores_enc_hostsim.cpp -- TEST INFRASTRUCTURE, NOT PRODUCT.
// The product's ProRes encoder (libav_b200/csrc/prores_enc.cu with prores_enc.cuh: every stage kernel, the checks and both entry points)
// compiled UNCHANGED as host C++: its kernels' threads never communicate, so running them one after the other encodes whole packets.
#include "shim/cuda_runtime.h"
#include "../../libav_b200/csrc/prores_enc.cu"

// the product's restated tables, in the order of ref_prores_enc_tables (oracle/refbuild/refapi_prores_enc.c): both scans, the DC and AC
// codebooks, run_to_cb_index, lev_to_cb_index, FIRST_DC_CB, the quantiser matrices, per profile min_quant / max_quant / br_tab[4], the
// macroblock limits.  Returns the count.
extern "C" int hostsim_prores_enc_tables(int32_t *out)
{
    using namespace avb;
    int n = 0;
    for (int s = 0; s < 2; s++) for (int i = 0; i < 64; i++) out[n++] = pe_scan[s][i];
    for (int i = 0; i < 4; i++) out[n++] = pe_dc_codebook[i];
    for (int i = 0; i < 7; i++) out[n++] = pe_ac_codebook[i];
    for (int i = 0; i < 16; i++) out[n++] = pe_run_to_cb[i];
    for (int i = 0; i < 10; i++) out[n++] = pe_lev_to_cb[i];
    out[n++] = PE_FIRST_DC_CB;
    for (int m = 0; m < 5; m++) for (int i = 0; i < 64; i++) out[n++] = pe_quant_matrices[m][i];
    for (int p = 0; p < 5; p++) {
        out[n++] = pe_profiles[p].min_quant; out[n++] = pe_profiles[p].max_quant;
        for (int i = 0; i < 4; i++) out[n++] = pe_profiles[p].br_tab[i];
    }
    for (int i = 0; i < 4; i++) out[n++] = pe_mb_limits[i];
    return n;
}
