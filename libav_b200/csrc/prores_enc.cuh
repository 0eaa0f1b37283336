// libav_b200/csrc/prores_enc.cuh -- the ProRes encoder's arithmetic (libavcodec/proresenc.c), device functions that the kernels of
// prores_enc.cu and their host build (tests/hostsim/) share: the slice grid, get_slice_data / get_alpha_data per block, prores_fdct,
// the rate-control estimates (estimate_dcs / estimate_acs / estimate_alpha_plane) and the entropy coder (encode_dcs / encode_acs /
// encode_alpha_plane) over a bit sink that either counts or writes MSB-first as put_bits / flush_put_bits do.
#pragma once
#include "common.cuh"
#include "fdct10.cuh"
#include "prores_tables.cuh"
#include <limits.h>

namespace avb {

constexpr int PE_SCORE_LIMIT = INT_MAX / 2;
constexpr int PE_NQ = 10;                  // trellis nodes per slice: min_quant..max_quant + 1 of the widest profile (LT: 1..10)

struct PeEst { int bits[PE_NQ]; int score[PE_NQ]; int overquant; };

// one frame as the kernels see it: encode_init's derivations (checked and filled on the host) and the frame's part of the workspace
struct PeFrame {
    const uint8_t *data[4];
    int ls[4];
    int width, height, c444, abits, ppf, tff;
    int mbw, mbh, mps, lmps, sw, spp, nslices;   // slices per row, per picture, per frame
    int minq, maxq, nq, bits_per_mb, force_quant, scan;
    uint8_t qm[64];
    uint8_t vendor[4], prim, trc, csp, matrix;
    int16_t *coef, *alpha;
    PeEst *est;
    int8_t *back;                               // nslices x PE_NQ trellis back-pointers
    int32_t *sq;                                // each slice's quantiser
    uint32_t *size;                             // nslices x 4 plane bytes
    uint32_t *off;                              // each slice's byte offset in the packet
    uint32_t *pic_size;                         // bytes of each picture
    uint8_t *out;
    size_t cap;
    int32_t *out_size;
};

__device__ inline int pe_log2(unsigned v)
{
#ifdef __CUDA_ARCH__
    return 31 - __clz(v);
#else
    return 31 - __builtin_clz(v);
#endif
}
__device__ inline int pe_make_code(int x) { return (int)((unsigned)x << 1) ^ (x >> 31); }
__device__ inline int pe_abs(int x) { return x < 0 ? -x : x; }

// ---- the slice grid: full slices of mbs_per_slice, then the set bits of the rest, largest first (the encoder halves mbs_per_slice at
// the right edge until the slice fits) ------------------------------------------------------------------------------------------------
__device__ inline void pe_slice_span(const PeFrame &F, int col, int &x0, int &mbs)
{
    const int full = F.mbw >> F.lmps;
    if (col < full) { x0 = col << F.lmps; mbs = F.mps; return; }
    x0 = full << F.lmps; mbs = 0;
    int k = col - full;
    for (int m = F.mps >> 1; m; m >>= 1) {
        if (!(F.mbw & m)) continue;
        if (!k) { mbs = m; return; }
        x0 += m; k--;
    }
}
// the slice holding macroblock column x: its column, first macroblock and width
__device__ inline int pe_slice_of_mb(const PeFrame &F, int x, int &x0, int &mbs)
{
    const int full = F.mbw >> F.lmps;
    if ((x >> F.lmps) < full) { x0 = (x >> F.lmps) << F.lmps; mbs = F.mps; return x >> F.lmps; }
    int col = full;
    x0 = full << F.lmps; mbs = 0;
    for (int m = F.mps >> 1; m; m >>= 1) {
        if (!(F.mbw & m)) continue;
        if (x < x0 + m) { mbs = m; return col; }
        x0 += m; col++;
    }
    return col;
}

struct PeSlice { const int16_t *blk[3]; const int16_t *alpha; int x0, mbs, nb[3]; };
// the staged coefficients of slice (pic, row, col): per plane the macroblocks in raster order, each macroblock's blocks in the encoder's
// order; alpha as get_alpha_data lays it out (16 lines of 16 * mbs samples)
__device__ inline PeSlice pe_slice(const PeFrame &F, int pic, int row, int col)
{
    PeSlice S;
    pe_slice_span(F, col, S.x0, S.mbs);
    const int ncb = F.c444 ? 4 : 2;
    const size_t mbs_pic = (size_t)F.mbw * F.mbh, m = (size_t)row * F.mbw + S.x0;
    const int16_t *base = F.coef + (size_t)pic * mbs_pic * (4 + 2 * ncb) * 64;
    S.blk[0] = base + m * 4 * 64;
    S.blk[1] = base + (mbs_pic * 4 + m * ncb) * 64;
    S.blk[2] = base + (mbs_pic * (4 + ncb) + m * ncb) * 64;
    S.alpha = F.alpha ? F.alpha + ((size_t)pic * mbs_pic + m) * 256 : nullptr;
    S.nb[0] = 4 * S.mbs; S.nb[1] = S.nb[2] = ncb * S.mbs;
    return S;
}

// ---- fetch: one 8 x 8 block as get_slice_data + prores_fdct leave it -----------------------------------------------------------------
// Edge emulation replicates the plane's last column, then its last line; both reduce to clamping the sample position.  A 4:2:2 chroma
// macroblock starting at or past width >> 1 is zero.  Fields read every other line from line_add = cur_picture_idx ^ !top_field_first, over
// height / pictures_per_frame lines.
__device__ inline int pe_plane_width(const PeFrame &F, int p) { return p == 1 || p == 2 ? (F.c444 ? F.width : F.width >> 1) : F.width; }
__device__ inline const uint16_t *pe_line(const PeFrame &F, int p, int pic, int line)
{
    const int line_add = F.ppf == 1 ? 0 : (pic ^ !F.tff);
    return reinterpret_cast<const uint16_t *>(F.data[p] + ((ptrdiff_t)line * F.ppf + line_add) * F.ls[p]);
}
__device__ inline void pe_fetch_fdct(const PeFrame &F, int pic, int p, int mby, int mbx, int b, int16_t *out)
{
    const bool sub = p && !F.c444;
    const int pw = pe_plane_width(F, p), h = F.height / F.ppf;
    const int xp = mbx << (sub ? 3 : 4), yp = mby << 4;
    if (xp >= pw) {
        for (int k = 0; k < 64; k++) out[k] = 0;
        return;
    }
    int dx, dy;
    if (p == 0) { dx = (b & 1) * 8; dy = (b >> 1) * 8; }           // TL TR BL BR
    else if (F.c444) { dx = (b >> 1) * 8; dy = (b & 1) * 8; }      // TL BL TR BR
    else { dx = 0; dy = b * 8; }                                    // top, bottom
    int16_t blk[64];
    for (int r = 0; r < 8; r++) {
        const uint16_t *src = pe_line(F, p, pic, min(yp + dy + r, h - 1));
        for (int c = 0; c < 8; c++) blk[8 * r + c] = (int16_t)src[min(xp + dx + c, pw - 1)];
    }
    int in[8], o[8];
    for (int r = 0; r < 8; r++) {                                   // ff_jpeg_fdct_islow_10: rows with int16 write-back, then columns
        for (int k = 0; k < 8; k++) in[k] = blk[8 * r + k];
        f10_islow_1d(in, o, 1, 12);
        for (int k = 0; k < 8; k++) blk[8 * r + k] = (int16_t)o[k];
    }
    for (int c = 0; c < 8; c++) {
        for (int k = 0; k < 8; k++) in[k] = blk[8 * k + c];
        f10_islow_1d(in, o, -2, 15);
        for (int k = 0; k < 8; k++) out[8 * k + c] = (int16_t)o[k];
    }
}
// get_alpha_data for one line of one macroblock: 16 samples, >> 2 at 8 bits, (v << 6) | (v >> 4) at 16 bits (int16 wrap)
__device__ inline void pe_fetch_alpha(const PeFrame &F, int pic, int mby, int mbx, int r, int16_t *out)
{
    const uint16_t *src = pe_line(F, 3, pic, min((mby << 4) + r, F.height / F.ppf - 1));
    for (int c = 0; c < 16; c++) {
        const int v = src[min((mbx << 4) + c, F.width - 1)];
        out[c] = (int16_t)(F.abits == 8 ? v >> 2 : (v << 6) | (v >> 4));
    }
}

// ---- estimates (find_slice_quant) ------------------------------------------------------------------------------------------------------
__device__ __forceinline__ int pe_vlc_len(unsigned codebook, int val)
{
    const unsigned switch_bits = (codebook & 3) + 1, rice_order = codebook >> 5, exp_order = (codebook >> 2) & 7;
    const unsigned switch_val = switch_bits << rice_order;
    if ((unsigned)val >= switch_val) {
        val -= switch_val - (1 << exp_order);
        return pe_log2((unsigned)val) * 2 - (int)exp_order + (int)switch_bits + 1;
    }
    return (val >> rice_order) + (int)rice_order + 1;
}
// estimate_dcs + estimate_acs of one plane, rounded up to bytes as estimate_slice_plane does.  The DC error starts at the SECOND block
// (estimate_dcs adds blocks[64]'s remainder before its loop, which adds it again)
__device__ __forceinline__ int pe_est_plane(int &error, const int16_t *blocks, int nb, const uint8_t *scan, const uint8_t *qm, int q)
{
    const int scale = qm[0] * q;
    int prev_dc = (blocks[0] - 0x4000) / scale;
    int bits = pe_vlc_len(PE_FIRST_DC_CB, pe_make_code(prev_dc));
    int sign = 0, codebook = 3;
    error += pe_abs(blocks[64] - 0x4000) % scale;
    for (int i = 1; i < nb; i++) {
        const int v = blocks[64 * i] - 0x4000, dc = v / scale;
        error += pe_abs(v) % scale;
        int delta = dc - prev_dc;
        const int new_sign = delta >> 31;
        delta = (delta ^ sign) - sign;
        const int code = pe_make_code(delta);
        bits += pe_vlc_len(pe_dc_codebook[codebook], code);
        codebook = min((code + (code & 1)) >> 1, 3);
        sign = new_sign;
        prev_dc = dc;
    }
    const int max_coeffs = nb << 6;
    int run_cb = pe_run_to_cb[4], lev_cb = pe_lev_to_cb[2], run = 0;
    for (int i = 1; i < 64; i++) {
        const int qv = qm[scan[i]] * q;
        for (int idx = scan[i]; idx < max_coeffs; idx += 64) {
            const int c = blocks[idx], level = c / qv;
            error += pe_abs(c) % qv;
            if (level) {
                const int abs_level = pe_abs(level);
                bits += pe_vlc_len(pe_ac_codebook[run_cb], run) + pe_vlc_len(pe_ac_codebook[lev_cb], abs_level - 1) + 1;
                run_cb = pe_run_to_cb[min(run, 15)];
                lev_cb = pe_lev_to_cb[min(abs_level, 9)];
                run = 0;
            } else run++;
        }
    }
    return (bits + 7) & ~7;
}
__device__ inline bool pe_alpha_long(int cur, int prev, int abits, int &diff)
{
    const int dsize = 1 << ((abits == 8 ? 4 : 7) - 1);
    diff = (cur - prev) & ((1 << abits) - 1);
    if (diff >= (1 << abits) - dsize) diff -= 1 << abits;
    return diff < -dsize || diff > dsize || !diff;
}
// estimate_alpha_plane: runs count 4 / 15 bits (put_alpha_run writes 5 / 16) and the total is not rounded to bytes
__device__ __forceinline__ int pe_est_alpha(const int16_t *a, int n, int abits)
{
    const int dbits = abits == 8 ? 4 : 7;
    int prev = (1 << abits) - 1, run = 0, diff;
    int cur = a[0];
    int bits = pe_alpha_long(cur, prev, abits, diff) ? abits + 1 : dbits + 1;
    prev = cur;
    for (int idx = 1; idx < n; idx++) {
        cur = a[idx];
        if (cur != prev) {
            bits += !run ? 1 : run < 0x10 ? 4 : 15;
            bits += pe_alpha_long(cur, prev, abits, diff) ? abits + 1 : dbits + 1;
            prev = cur;
            run = 0;
        } else run++;
    }
    if (run) bits += run < 0x10 ? 4 : 15;
    return bits;
}
// one slice at quantiser q: bits and error over every plane.  estimate_alpha_plane sets the error to 0, so with alpha it is 0
__device__ inline int pe_est_slice(const PeFrame &F, const PeSlice &S, int q, int &error)
{
    error = 0;
    int bits = 0;
#pragma unroll
    for (int p = 0; p < 3; p++) bits += pe_est_plane(error, S.blk[p], S.nb[p], pe_scan[F.scan], F.qm, q);
    if (F.abits) {
        bits += pe_est_alpha(S.alpha, S.mbs * 256, F.abits);
        error = 0;
    }
    return bits;
}

// ---- the entropy coder over a bit sink --------------------------------------------------------------------------------------------------
struct PeCount {
    long long bits = 0;
    __device__ void put(int n, unsigned) { bits += n; }
};
// put_bits MSB-first into bytes; flush() pads the last byte with zeros, as flush_put_bits does
struct PeWriter {
    uint8_t *p;
    unsigned long long acc = 0;
    int n = 0;
    __device__ explicit PeWriter(uint8_t *dst) : p(dst) {}
    __device__ void put(int bits, unsigned v)
    {
        if (!bits) return;
        acc = (acc << bits) | v;
        n += bits;
        while (n >= 8) { n -= 8; *p++ = (uint8_t)(acc >> n); }
    }
    __device__ void flush() { if (n) { *p++ = (uint8_t)(acc << (8 - n)); n = 0; } }
};
template <class S> __device__ inline void pe_put_vlc(S &pb, unsigned codebook, int val)
{
    const unsigned switch_bits = (codebook & 3) + 1, rice_order = codebook >> 5, exp_order = (codebook >> 2) & 7;
    const unsigned switch_val = switch_bits << rice_order;
    if ((unsigned)val >= switch_val) {
        val -= switch_val - (1 << exp_order);
        const int exponent = pe_log2((unsigned)val);
        pb.put(exponent - (int)exp_order + (int)switch_bits, 0);
        pb.put(exponent + 1, (unsigned)val);
    } else {
        const int exponent = val >> rice_order;
        if (exponent) pb.put(exponent, 0);
        pb.put(1, 1);
        if (rice_order) pb.put((int)rice_order, (unsigned)val & ((1u << rice_order) - 1));
    }
}
// encode_dcs + encode_acs of one plane
template <class S> __device__ inline void pe_code_plane(S &pb, const int16_t *blocks, int nb, const uint8_t *scan, const uint8_t *qm, int q)
{
    const int scale = qm[0] * q;
    int prev_dc = (blocks[0] - 0x4000) / scale;
    pe_put_vlc(pb, PE_FIRST_DC_CB, pe_make_code(prev_dc));
    int sign = 0, codebook = 3;
    for (int i = 1; i < nb; i++) {
        const int dc = (blocks[64 * i] - 0x4000) / scale;
        int delta = dc - prev_dc;
        const int new_sign = delta >> 31;
        delta = (delta ^ sign) - sign;
        const int code = pe_make_code(delta);
        pe_put_vlc(pb, pe_dc_codebook[codebook], code);
        codebook = min((code + (code & 1)) >> 1, 3);
        sign = new_sign;
        prev_dc = dc;
    }
    const int max_coeffs = nb << 6;
    int run_cb = pe_run_to_cb[4], lev_cb = pe_lev_to_cb[2], run = 0;
    for (int i = 1; i < 64; i++) {
        const int qv = qm[scan[i]] * q;
        for (int idx = scan[i]; idx < max_coeffs; idx += 64) {
            const int level = blocks[idx] / qv;
            if (level) {
                const int abs_level = pe_abs(level);
                pe_put_vlc(pb, pe_ac_codebook[run_cb], run);
                pe_put_vlc(pb, pe_ac_codebook[lev_cb], abs_level - 1);
                pb.put(1, level < 0);
                run_cb = pe_run_to_cb[min(run, 15)];
                lev_cb = pe_lev_to_cb[min(abs_level, 9)];
                run = 0;
            } else run++;
        }
    }
}
template <class S> __device__ inline void pe_put_alpha_diff(S &pb, int cur, int prev, int abits)
{
    const int dbits = abits == 8 ? 4 : 7;
    int diff;
    if (pe_alpha_long(cur, prev, abits, diff)) { pb.put(1, 1); pb.put(abits, (unsigned)diff); }
    else { pb.put(1, 0); pb.put(dbits - 1, (unsigned)(pe_abs(diff) - 1)); pb.put(1, diff < 0); }
}
template <class S> __device__ inline void pe_put_alpha_run(S &pb, int run)
{
    if (run) { pb.put(1, 0); pb.put(run < 0x10 ? 4 : 15, (unsigned)run); }
    else pb.put(1, 1);
}
// encode_alpha_plane (it reads the samples as uint16_t)
template <class S> __device__ inline void pe_code_alpha(S &pb, const int16_t *a, int n, int abits)
{
    int prev = (1 << abits) - 1, run = 0;
    int cur = (uint16_t)a[0];
    pe_put_alpha_diff(pb, cur, prev, abits);
    prev = cur;
    for (int idx = 1; idx < n; idx++) {
        cur = (uint16_t)a[idx];
        if (cur != prev) {
            pe_put_alpha_run(pb, run);
            pe_put_alpha_diff(pb, cur, prev, abits);
            prev = cur;
            run = 0;
        } else run++;
    }
    if (run) pe_put_alpha_run(pb, run);
}
// plane p of a slice at quantiser q through a sink
template <class S> __device__ inline void pe_code_slice_plane(S &pb, const PeFrame &F, const PeSlice &sl, int p, int q)
{
    if (p < 3) pe_code_plane(pb, sl.blk[p], sl.nb[p], pe_scan[F.scan], F.qm, q);
    else pe_code_alpha(pb, sl.alpha, sl.mbs * 256, F.abits);
}

}  // namespace avb
