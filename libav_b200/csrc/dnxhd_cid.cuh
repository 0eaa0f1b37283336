// libav_b200/csrc/dnxhd_cid.cuh -- host code that the VC-3 / DNxHD encoder (dnxhd_enc.cu) and decoder (dnxhd_dec.cu) share: a checksum of
// the arrays of a caller's CID entry (FFDnxhdCidEntry) and a cache of the device tables each codec builds from an entry, keyed by the
// entry's host address and rebuilt when its checksum changes.  Each including file keeps its own cache for its own table type.
#pragma once
#include "common.cuh"
#include "../../include/avdsp_b200.h"
#include <map>
#include <mutex>
#include <vector>

namespace avb {
namespace {

// the arrays of an entry that the tables are built from, and how many of each (dc: bit_depth + 4 codes, ac: 257, run: 62)
uint64_t dn_checksum(const FFDnxhdCidEntry &e)
{
    uint64_t h = 0xcbf29ce484222325ull;
    auto mix = [&](const void *p, size_t n) {
        const uint8_t *b = (const uint8_t *)p;
        for (size_t k = 0; k < n; k++) h = (h ^ b[k]) * 0x100000001b3ull;
    };
    mix(&e.cid, 8 * sizeof(int));
    const size_t ndc = (size_t)e.bit_depth + 4;
    mix(e.luma_weight, 64); mix(e.chroma_weight, 64); mix(e.dc_codes, ndc); mix(e.dc_bits, ndc);
    mix(e.ac_codes, 257 * 2); mix(e.ac_bits, 257); mix(e.ac_level, 257); mix(e.ac_run_flag, 257); mix(e.ac_index_flag, 257);
    mix(e.run_codes, 62 * 2); mix(e.run_bits, 62); mix(e.run, 62);
    return h;
}

// the device tables T of an entry, built on the host by build(entry, T) (0, or -1 with a message set) on the first call for an address
// and whenever the entry's checksum changes; the old copy stays alive, because a launch still queued may read it.  `where` names the
// caller in error messages.
template <class T, class Build> const T *dn_tables_cached(const FFDnxhdCidEntry *e, Build build, const char *where)
{
    struct Cached { T *d; uint64_t sum; };
    static std::mutex mu;
    static std::map<const FFDnxhdCidEntry *, Cached> cache;
    const uint64_t sum = dn_checksum(*e);
    std::lock_guard<std::mutex> lk(mu);
    auto it = cache.find(e);
    if (it != cache.end() && it->second.sum == sum) return it->second.d;
    std::vector<uint8_t> host(sizeof(T));
    T &t = *reinterpret_cast<T *>(host.data());
    if (build(*e, t)) return nullptr;
    T *d = nullptr;
    if (cudaMalloc(&d, sizeof(T)) != cudaSuccess) { set_error(where, cudaGetLastError()); return nullptr; }
    if (cudaMemcpy(d, &t, sizeof(T), cudaMemcpyHostToDevice) != cudaSuccess) {
        set_error(where, cudaGetLastError());
        cudaFree(d);
        return nullptr;
    }
    cache[e] = Cached{ d, sum };
    return d;
}

}  // namespace
}  // namespace avb
