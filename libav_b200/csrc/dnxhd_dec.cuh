// libav_b200/csrc/dnxhd_dec.cuh -- the VC-3 / DNxHD decoder's arithmetic (libavcodec/dnxhddec.c), device functions that the kernels of
// dnxhd_dec.cu and their host build (tests/hostsim/) share: the bit reader (the packet, then zero bits), the two-level VLC lookups, one
// macroblock row's entropy decoding and dequantisation (dnxhd_decode_macroblock's bitstream half and dnxhd_decode_dct_block), and one
// block's ff_simple_idct_put_8 / ff_simple_idct_put_10 at the place dnxhd_decode_macroblock puts it.
#pragma once
#include "common.cuh"
#include "idct10.cuh"
#include "simple_idct8.cuh"

namespace avb {

constexpr int DD_VLC_BITS = 9;                   // first level of the AC and run lookups; a second level of 7 bits reaches 16-bit codes
constexpr int DD_SUB_BITS = 7;
constexpr int DD_AC_N = 512 + 128 * 24;          // first level + up to 24 second-level tables (the CIDs of dnxhddata.c need 14)
constexpr int DD_RUN_N = 512 + 128 * 32;         // (they need 24)
constexpr int DD_MAX_ROWS = 68;                  // mb_scan_index[68]

// The lookup tables of a CID entry, built on the host (dnxhd_dec.cu) and staged in shared memory by each CTA of the entropy stage.
// ac / run entries: bit 15 set: a second-level table at (entry & 0x7fff), indexed by the next 7 bits.  Otherwise a leaf: bits 0..4 the
// code's whole length, bits 5..14 the payload: for ac the level (ac_level, 8 bits), the index flag (bit 13) and the run flag (bit 14);
// for run the run (8 bits).  dc: bits 0..2 the code's length, bits 3..6 the symbol (the count of difference bits).
struct DdTables {
    uint16_t ac[DD_AC_N];
    uint16_t run[DD_RUN_N];
    uint8_t dc[128];
    uint8_t weight[2][64];                       // luma, chroma, in scan order
    uint8_t zz[64];                              // ff_zigzag_direct (FF_IDCT_PERM_NONE for both IDCTs)
};

struct DdUnit { uint32_t off; int mbh, mbaff, cur_field; };   // a coding unit: its byte offset in the packet and its header's fields

// one packet as the kernels see it: what the header checks derived on the host, and its part of the workspace
struct DdFrame {
    const uint8_t *pkt;
    uint8_t *data[3];
    const DdTables *tab;
    int16_t *coef;                               // per row of each unit in turn: mbw macroblocks x nblk blocks x 64 coefficients
    uint8_t *ilmb;                               // per row of each unit: each macroblock's interlaced_mb
    uint32_t size;
    int ls[3];
    int mbw, nu, rows, bd10, is444, il, gray;
    DdUnit u[2];
};

__host__ __device__ inline uint32_t dd_be32(const uint8_t *p) { return (uint32_t)p[0] << 24 | (uint32_t)p[1] << 16 | (uint32_t)p[2] << 8 | p[3]; }

// ---- the bit reader: bytes [0, size) of the packet, then zero bits -----------------------------------------------------------------------
// Words are loaded at 4-byte-aligned addresses; a word is loaded only when it holds a byte of the packet, and its bytes past the end are
// cleared.  After refill() at least 33 bits are valid.
struct DdBits {
    const uint8_t *abase;                        // the packet's address rounded down to 4 bytes
    uint32_t end, w;                             // the packet's end and the next word, as offsets from abase
    uint64_t cache;                              // valid bits MSB-first
    int n;
};
__device__ __forceinline__ uint32_t dd_word(const DdBits &r, uint32_t w)
{
    if (w >= r.end) return 0;
    uint32_t v = *reinterpret_cast<const uint32_t *>(r.abase + w);
#ifdef __CUDA_ARCH__
    v = __byte_perm(v, 0, 0x0123);
#else
    v = __builtin_bswap32(v);
#endif
    const uint32_t left = r.end - w;
    return left >= 4 ? v : v & ~(0xffffffffu >> (8 * left));
}
__device__ __forceinline__ void dd_refill(DdBits &r)
{
    if (r.n <= 32) { r.cache |= (uint64_t)dd_word(r, r.w) << (32 - r.n); r.n += 32; r.w += 4; }
}
__device__ __forceinline__ void dd_bits_init(DdBits &r, const uint8_t *pkt, uint32_t size, uint32_t start)
{
    const uint32_t mis = (uint32_t)((uintptr_t)pkt & 3);
    r.abase = pkt - mis;
    r.end = size + mis;
    const uint32_t o = start + mis;
    r.w = o & ~3u;
    r.cache = 0; r.n = 0;
    dd_refill(r);
    const int drop = 8 * (int)(o & 3);
    r.cache <<= drop; r.n -= drop;
    dd_refill(r);
}
__device__ __forceinline__ uint32_t dd_peek(const DdBits &r, int k) { return (uint32_t)(r.cache >> (64 - k)); }      // 1 <= k <= 32
__device__ __forceinline__ void dd_skip(DdBits &r, int k) { r.cache <<= k; r.n -= k; }
__device__ __forceinline__ uint32_t dd_get(DdBits &r, int k) { const uint32_t v = dd_peek(r, k); dd_skip(r, k); return v; }

// a leaf of a two-level table (the code is consumed)
__device__ __forceinline__ unsigned dd_vlc(DdBits &r, const uint16_t *t)
{
    unsigned e = t[dd_peek(r, DD_VLC_BITS)];
    if (e & 0x8000u) e = t[(e & 0x7fffu) + (dd_peek(r, DD_VLC_BITS + DD_SUB_BITS) & ((1u << DD_SUB_BITS) - 1))];
    dd_skip(r, (int)(e & 31));
    return e >> 5;
}

// ---- entropy: one macroblock row of a coding unit --------------------------------------------------------------------------------------
// dnxhd_decode_dct_block with the decoder's (index_bits, level_bias, level_shift): (4, 32, 6) at 8 bit, (6, 8, 4) at 10-bit 4:2:2,
// (6, 32, 6) at 4:4:4.  blk holds 64 zeros on entry.
template <int IB, int BIAS, int SH>
__device__ inline void dd_block(DdBits &r, const DdTables &T, int16_t *blk, int &last_dc, const uint8_t *weight, unsigned qscale)
{
    dd_refill(r);
    const unsigned d = T.dc[dd_peek(r, 7)];
    dd_skip(r, (int)(d & 7));
    const int len = (int)(d >> 3);
    if (len) {
        const int top = (int)(r.cache >> 63);
        const int b = (int)dd_get(r, len);
        last_dc = (int)((unsigned)last_dc + (unsigned)(top ? b : b - ((1 << len) - 1)));
    }
    blk[0] = (int16_t)last_dc;
    for (int i = 1;; i++) {
        dd_refill(r);
        const unsigned e = dd_vlc(r, T.ac);
        int level = (int)(e & 255);
        if (!level) break;                                                   // EOB
        const unsigned sign = 0u - dd_get(r, 1);
        if (e & 0x100u) level += (int)dd_get(r, IB) << 6;
        if (e & 0x200u) {
            dd_refill(r);
            i += (int)(dd_vlc(r, T.run) & 255);
        }
        if (i > 63) break;                                                   // "ac tex damaged": the next block starts here
        const unsigned w = weight[i];
        unsigned v = (unsigned)(2 * level + 1) * qscale * w;                 // 32-bit wrap-around, as the C int arithmetic
        if (BIAS < 32 || w != (unsigned)BIAS) v += BIAS;
        const int lv = (int)v >> SH;
        blk[T.zz[i]] = (int16_t)(((unsigned)lv ^ sign) - sign);
    }
}

template <int IB, int BIAS, int SH, bool I444>
__device__ inline void dd_row_t(const DdFrame &F, const DdTables &T, int unit, int y, int16_t *coef, uint8_t *ilmb)
{
    const DdUnit &U = F.u[unit];
    const uint32_t scan = dd_be32(F.pkt + U.off + 0x170 + 4 * y);
    DdBits r;
    dd_bits_init(r, F.pkt, F.size, U.off + 0x280 + scan);
    int last_dc[3];
    last_dc[0] = last_dc[1] = last_dc[2] = 1 << (F.bd10 ? 12 : 10);
    constexpr int NB = I444 ? 12 : 8;
    for (int x = 0; x < F.mbw; x++) {
        dd_refill(r);
        unsigned il = 0, qscale;
        if (U.mbaff) { il = dd_get(r, 1); qscale = dd_get(r, 10); }
        else qscale = dd_get(r, 11);
        dd_skip(r, 1);
        ilmb[x] = (uint8_t)il;
        for (int n = 0; n < NB; n++) {
            int16_t *blk = coef + ((size_t)x * NB + n) * 64;
            uint4 *b4 = reinterpret_cast<uint4 *>(blk);
            for (int k = 0; k < 8; k++) b4[k] = make_uint4(0, 0, 0, 0);
            int comp;
            if (!I444) comp = n & 2 ? 1 + (n & 1) : 0;
            else comp = (n >> 1) % 3;
            dd_block<IB, BIAS, SH>(r, T, blk, last_dc[comp], T.weight[comp ? 1 : 0], qscale);
        }
    }
}
// row t of the packet (the first unit's rows, then the second's)
__device__ inline void dd_row(const DdFrame &F, const DdTables &T, int t)
{
    const int unit = t >= F.u[0].mbh, y = unit ? t - F.u[0].mbh : t;
    const int nb = F.is444 ? 12 : 8;
    int16_t *coef = F.coef + (size_t)t * F.mbw * nb * 64;
    uint8_t *ilmb = F.ilmb + (size_t)t * F.mbw;
    if (!F.bd10) dd_row_t<4, 32, 6, false>(F, T, unit, y, coef, ilmb);
    else if (!F.is444) dd_row_t<6, 8, 4, false>(F, T, unit, y, coef, ilmb);
    else dd_row_t<6, 32, 6, true>(F, T, unit, y, coef, ilmb);
}

// ---- reconstruction: block b of macroblock mb of row t ------------------------------------------------------------------------------------
// idct_put at the destination and line step dnxhd_decode_macroblock gives the block.  Returns without writing for chroma under gray.
__device__ inline void dd_put_block(const DdFrame &F, int t, int mb, int b)
{
    const int unit = t >= F.u[0].mbh, y = unit ? t - F.u[0].mbh : t, x = mb;
    const DdUnit &U = F.u[unit];
    const int nb = F.is444 ? 12 : 8, shift1 = F.bd10;
    // plane, column (0 / 1) and row (0 / 1) of the block in its macroblock
    int plane, cx, cy;
    if (!F.is444) {
        static constexpr uint8_t P[8] = { 0, 0, 1, 2, 0, 0, 1, 2 }, X[8] = { 0, 1, 0, 0, 0, 1, 0, 0 };
        plane = P[b]; cx = X[b]; cy = b >= 4;
    } else {
        static constexpr uint8_t P[12] = { 0, 0, 1, 1, 2, 2, 0, 0, 1, 1, 2, 2 };
        plane = P[b]; cx = b & 1; cy = b >= 6;
    }
    if (plane && F.gray) return;
    const int il = F.ilmb[(size_t)t * F.mbw + mb];
    const ptrdiff_t ls = F.ls[plane ? 1 : 0];                                  // V is stepped with U's linesize, as the reference does
    ptrdiff_t dls = ls << F.il;
    uint8_t *dest = F.data[plane] + ((ptrdiff_t)y * dls << 4) + ((ptrdiff_t)x << (plane && !F.is444 ? 3 + shift1 : 4 + shift1));
    if (U.cur_field) dest += F.ls[plane];
    if (il) dls <<= 1;
    const ptrdiff_t yoff = il ? ls : dls << 3;
    dest += cx * (8 << shift1) + cy * yoff;

    alignas(16) int16_t blk[64];
    const uint4 *src = reinterpret_cast<const uint4 *>(F.coef + (((size_t)t * F.mbw + mb) * nb + b) * 64);
    uint4 *b4 = reinterpret_cast<uint4 *>(blk);
    for (int k = 0; k < 8; k++) b4[k] = src[k];
    if (!shift1) {                                                             // ff_simple_idct_put_8
        enc_idct_rows(blk);
        for (int c = 0; c < 8; c++) {
            int o[8];
            enc_idct_col(blk + c, o);
            for (int k = 0; k < 8; k++) dest[k * dls + c] = (uint8_t)min(max(o[k], 0), 255);
        }
        return;
    }
    for (int k = 0; k < 8; k++) b4[k] = i10_row(b4[k]);                        // ff_simple_idct_put_10
    for (int c = 0; c < 8; c++) {
        uint32_t w[8];
        for (int k = 0; k < 8; k++) {
            const uint4 v = b4[k];
            w[k] = (c >> 1) == 0 ? v.x : (c >> 1) == 1 ? v.y : (c >> 1) == 2 ? v.z : v.w;
        }
        int o[8];
        if (c & 1) i10_col<1>(w, o); else i10_col<0>(w, o);
        for (int k = 0; k < 8; k++) reinterpret_cast<uint16_t *>(dest + k * dls)[c] = (uint16_t)i10_clip(o[k]);
    }
}

}  // namespace avb
