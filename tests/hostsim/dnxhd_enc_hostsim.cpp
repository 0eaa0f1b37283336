// tests/hostsim/dnxhd_enc_hostsim.cpp -- TEST INFRASTRUCTURE, NOT PRODUCT.
// The product's DNxHD encoder (libav_b200/csrc/dnxhd_enc.cu with dnxhd_enc.cuh: every stage kernel, the checks and both entry points)
// compiled UNCHANGED as host C++.  Its per-thread stages run one thread after the other; the rate-control search is launched with one thread
// per CTA here (DN_SEARCH_THREADS), for which its barriers are skipped, so the suite runs the product's own search code.
#include "shim/cuda_runtime.h"
#include "../../libav_b200/csrc/dnxhd_enc.cu"

// the tables the product builds from a CID entry (dnxhd_init_vlc), laid out as ref_dnxhd_vlc returns the reference's; returns max_level,
// or -1 when the entry is refused
extern "C" int hostsim_dnxhd_vlc(const FFDnxhdCidEntry *e, uint32_t *codes, uint8_t *bits, uint16_t *run_codes, uint8_t *run_bits)
{
    using namespace avb;
    std::vector<uint8_t> host(sizeof(DnTables));
    DnTables &T = *reinterpret_cast<DnTables *>(host.data());
    if (dn_build_tables(*e, T)) return -1;
    for (int i = 0; i < 4 * T.max_level; i++) { codes[i] = T.vlc_codes[i]; bits[i] = T.vlc_bits[i]; }
    for (int i = 0; i < 63; i++) { run_codes[i] = T.run_codes[i]; run_bits[i] = T.run_bits[i]; }
    return T.max_level;
}
