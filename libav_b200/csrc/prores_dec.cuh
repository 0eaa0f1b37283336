// libav_b200/csrc/prores_dec.cuh -- the ProRes decoder's entropy arithmetic (libavcodec/proresdec.c), device functions that the kernels of
// prores_dec.cu and their host build (tests/hostsim/) share: the checked long bitstream reader over one slice plane, decode_vlc_codeword,
// decode_dc_coeffs, decode_ac_coeffs, unpack_alpha and decode_slice's header parsing.
#pragma once
#include "common.cuh"
#include "prores_tables.cuh"
#include "prores.cuh"

namespace avb {

constexpr int PRD_CHUNK = 32;                    // slices per chunk of the slice-offset scan

// one picture of a packet (decode_picture_header's results, checked on the host) and its part of the workspace
struct PrdPic {
    uint32_t index;                              // packet offset of the picture's slice size table (be16 per slice)
    int n_slices, swf;
    int field;                                   // 1: the picture's lines start one frame line down
    uint32_t *chunks;                            // sums of PRD_CHUNK consecutive slice sizes
    uint32_t *offs;                              // n_slices + 1 slice offsets from the first slice (index + 2 n_slices)
    FFProresSlice *slices;
    uint32_t *status;                            // per slice: byte p = 1 when plane p's coefficients decoded (prores.cuh)
    int16_t *coef;                               // per slice: its Y, U and V blocks, in the order of ff_prores_decode_pictures_cuda
};

// one packet as the kernels see it
struct PrdFrame {
    const uint8_t *pkt;
    uint32_t size;
    int mbw, mbh;                                // num_x_mbs, num_y_mbs
    int c444, alpha;                             // chroma_factor 3; alpha_info of a format with alpha (1: 8-bit, 2: 16-bit), else 0
    int il, scan;                                // interlaced; the scan (0 progressive, 1 interlaced)
    int npics;
    uint8_t *adata;                              // the alpha plane and its frame linesize
    int als;
    PrdPic pic[2];
};

__host__ __device__ __forceinline__ int prd_bpm(int c444) { return c444 ? 12 : 8; }          // blocks per macroblock, Y + U + V

// slice s of a picture: its first macroblock column and width (decode_picture's loop)
__host__ __device__ inline void prd_slice_pos(int mbw, int swf, int nxs, int s, int &row, int &x, int &w)
{
    row = s / nxs;
    const int sc = s - row * nxs, full = mbw >> swf;
    if (sc < full) { x = sc << swf; w = 1 << swf; return; }
    x = full << swf; w = 0;                                           // the right edge: the set bits of the remainder, largest first
    int k = sc - full;
    for (int b = 2; b >= 0; b--) {
        if (!((mbw >> b) & 1) || b >= swf) continue;
        if (k == 0) { w = 1 << b; return; }
        x += 1 << b; k--;
    }
}

// ---- the checked long reader (get_bits.h with LONG_BITSTREAM_READER, UNCHECKED_BITSTREAM_READER 0) over one slice plane ---------------
// The position counts bits from the plane's first byte and stops at the plane's bits + 8.  Bytes past the plane are the packet's following
// bytes, bytes past the packet are zero (its padding).  The 32-bit cache at the clamp position reaches 5 bytes past the plane at most.
struct PrdBits {
    const uint8_t *pkt;
    uint32_t end;                                // the packet's size
    uint32_t start;                              // the plane's first byte
    int bits;                                    // size_in_bits
    int idx;                                     // index
};
__device__ __forceinline__ uint32_t prd_byte(const uint8_t *pkt, uint32_t end, uint32_t o) { return o < end ? pkt[o] : 0u; }
__device__ __forceinline__ void prd_bits_init(PrdBits &r, const PrdFrame &F, uint32_t start, int bytes)
{
    r.pkt = F.pkt; r.end = F.size; r.start = start; r.bits = bytes << 3; r.idx = 0;
}
// UPDATE_CACHE + GET_CACHE: the 32 bits at the position
__device__ __forceinline__ uint32_t prd_show32(const PrdBits &r)
{
    const uint32_t o = r.start + ((uint32_t)r.idx >> 3);
    uint64_t v = 0;
#pragma unroll
    for (int k = 0; k < 5; k++) v = v << 8 | prd_byte(r.pkt, r.end, o + k);
    return (uint32_t)(v >> (8 - (r.idx & 7)));
}
// SKIP_COUNTER of the checked reader
__device__ __forceinline__ void prd_skip(PrdBits &r, int n) { r.idx = min(r.bits + 8, r.idx + n); }
__device__ __forceinline__ uint32_t prd_get(PrdBits &r, int n) { const uint32_t v = prd_show32(r) >> (32 - n); prd_skip(r, n); return v; }
__device__ __forceinline__ int prd_clz(uint32_t v)                    // 31 - av_log2(v): 31 for 0
{
#ifdef __CUDA_ARCH__
    return __clz(v | 1);
#else
    return __builtin_clz(v | 1);
#endif
}

// decode_vlc_codeword
__device__ __forceinline__ uint32_t prd_vlc(PrdBits &r, unsigned cb)
{
    const uint32_t buf = prd_show32(r);
    const unsigned sw = (cb & 3) + 1, rice = cb >> 5, ex = (cb >> 2) & 7;
    const unsigned lg = (unsigned)prd_clz(buf);
    uint32_t code;
    int n;
    if (lg < sw) {
        if (!rice) { code = lg; n = (int)lg + 1; }
        else { code = (lg << rice) + ((buf << (lg + 1)) >> (32 - rice)); n = (int)(lg + 1 + rice); }
    } else {
        const unsigned len = 2 * lg - sw + ex + 1;
        // NEG_USR32(buf, len) is buf >> (32 - len), a negative count for len > 32 (a run of zero bits: FIRST_DC_CB with 31 leading zeros
        // gives 68), which C leaves undefined.  The reference as compiled for x86-64 shifts by the count modulo 32; CUDA's >> would give 0.
        code = (buf >> ((32 - len) & 31)) - (1u << ex) + (sw << rice);
        n = (int)len;
    }
    prd_skip(r, n);
    return code;
}

// decode_dc_coeffs: the DC of each of the plane's n blocks (blk: its first block)
__device__ inline void prd_dc(PrdBits &r, int16_t *blk, int n)
{
    uint32_t code = prd_vlc(r, PE_FIRST_DC_CB);
    int16_t prev = (int16_t)((code >> 1) ^ (0u - (code & 1)));
    blk[0] = prev;
    int16_t delta = 3;
    for (int i = 1; i < n; i++) {
        const int ad = delta < 0 ? -delta : delta;
        code = prd_vlc(r, pe_dc_codebook[ad < 3 ? ad : 3]);
        const uint32_t sign = 0u - (((uint32_t)(delta >> 15) & 1u) ^ (code & 1u));
        delta = (int16_t)((((code + 1) >> 1) ^ sign) - sign);
        prev = (int16_t)(prev + delta);
        blk[64 * i] = prev;
    }
}

// get_bits_left(gb) <= 0 || (get_bits_left(gb) <= MAX_PADDING && !show_bits(gb, get_bits_left(gb)))
__device__ __forceinline__ bool prd_exhausted(const PrdBits &r)
{
    const int left = r.bits - r.idx;
    return left <= 0 || (left <= 16 && !(prd_show32(r) >> (32 - left)));
}

// decode_ac_coeffs: 0, or -1 for AVERROR_INVALIDDATA
__device__ inline int prd_ac(PrdBits &r, int16_t *blk, int nblocks, int psf, const uint8_t *scan)
{
    int run = 4, level = 2;
    const int max_coeffs = nblocks << 6, mask = nblocks - 1;
    for (int pos = nblocks - 1; pos < max_coeffs;) {
        const int run_cb = pe_run_to_cb[min(run, 15)], lev_cb = pe_lev_to_cb[min(level, 9)];
        if (prd_exhausted(r)) return 0;
        run = (int)prd_vlc(r, pe_ac_codebook[run_cb]);
        if (run < 0) return -1;
        if (prd_exhausted(r)) return -1;
        level = (int)(prd_vlc(r, pe_ac_codebook[lev_cb]) + 1u);
        if (level < 0) return -1;
        pos += run + 1;
        if (pos >= max_coeffs) break;
        const int sign = (int)prd_show32(r) >> 31;                   // get_sbits(gb, 1)
        prd_skip(r, 1);
        blk[((pos & mask) << 6) + scan[pos >> psf]] = (int16_t)((level ^ sign) - sign);
    }
    return 0;
}

// unpack_alpha + decode_alpha_plane's copy: every sample of the slice's 16 lines of 16 * mbs samples, straight into the plane
template <int NB>
__device__ inline void prd_alpha(PrdBits &r, uint8_t *dst, ptrdiff_t ls, int mbs)
{
    const int mask = (1 << NB) - 1, num = mbs * 256, w = 16 * mbs;
    int idx = 0, alpha = mask;
    auto put = [&](int n) {
        const uint16_t v = (uint16_t)(NB == 16 ? alpha >> 6 : (alpha << 2) | (alpha >> 6));
        for (int i = 0; i < n; i++, idx++) {
            const int y = idx / w;
            reinterpret_cast<uint16_t *>(dst + y * ls)[idx - y * w] = v;
        }
    };
    do {
        do {
            int val;
            if (prd_get(r, 1)) val = (int)prd_get(r, NB);
            else {
                val = (int)prd_get(r, NB == 16 ? 7 : 4);
                const int sign = val & 1;
                val = (val + 2) >> 1;
                if (sign) val = -val;
            }
            alpha = (alpha + val) & mask;
            put(1);
            if (idx >= num - 1) break;
        } while (prd_get(r, 1));
        int val = (int)prd_get(r, 4);
        if (!val) val = (int)prd_get(r, 11);
        if (idx + val > num) val = num - idx;
        put(val);
    } while (idx < num);
}

// decode_slice's header: false for a slice that writes nothing (under 6 bytes, or sizes that do not fit); else the planes' offsets from
// the slice's first byte, their sizes (Y, U, V, alpha) and the scale factor
__device__ inline bool prd_slice_header(const PrdFrame &F, uint32_t off, int size, int coff[4], int sz[4], int &sf)
{
    if (size < 6) return false;
    uint32_t b[8];
#pragma unroll
    for (int k = 0; k < 8; k++) b[k] = prd_byte(F.pkt, F.size, off + k);
    const int hdr = (int)(b[0] >> 3);
    sz[0] = (int)(b[2] << 8 | b[3]);
    sz[1] = (int)(b[4] << 8 | b[5]);
    coff[0] = hdr;
    coff[1] = coff[0] + sz[0];
    coff[2] = coff[1] + sz[1];
    sz[2] = hdr > 7 ? (int)(b[6] << 8 | b[7]) : size - coff[2];
    coff[3] = coff[2] + sz[2];
    sz[3] = size - coff[3];
    if (sz[2] < 0 || sz[3] < 0 || hdr < 6) return false;
    sf = b[1] < 1 ? 1 : b[1] > 224 ? 224 : (int)b[1];
    sf = sf > 128 ? (sf - 96) << 2 : sf;
    return true;
}

}  // namespace avb
