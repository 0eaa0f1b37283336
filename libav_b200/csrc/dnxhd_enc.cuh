// libav_b200/csrc/dnxhd_enc.cuh -- the VC-3 / DNxHD encoder's arithmetic (libavcodec/dnxhdenc.c), device functions that the kernels of
// dnxhd_enc.cu and their host build (tests/hostsim/) share: the block fetch of dnxhd_get_blocks with the forward DCT, the quantisers
// (ff_dct_quantize_c at 8 bit, dnxhd_10bit_dct_quantize), the bit counts of dnxhd_calc_bits_thread with dnxhd_unquantize_c + IDCT + SSD
// for the RD rate control, the macroblock variance of dnxhd_mb_var_thread, and the coder of dnxhd_encode_thread over a bit sink.
#pragma once
#include "common.cuh"
#include "fdct_dev.cuh"
#include "fdct10.cuh"
#include "idct10.cuh"
#include "mpv_quant.cuh"
#include "simple_idct8.cuh"

namespace avb {

constexpr int DN_MAX_LEVEL = 1 << 12;            // 1 << (bit_depth + 2) at 10 bit; the VLC tables hold levels -max_level..max_level - 1
constexpr int DN_VLC_N = 4 * DN_MAX_LEVEL;
constexpr int DN_QMAX = 69;
constexpr int DN_EINVAL = -22;                   // AVERROR(EINVAL)
constexpr int DN_LAMBDA_FRAC_BITS = 10;
constexpr int DN_MAX_ROWS = 68;                  // macroblock rows of a 1080-line progressive picture

// what dnxhd_init_vlc / dnxhd_init_qmat build from a CID entry, on the device (built on the host by dnxhd_enc.cu)
struct DnTables {
    uint32_t vlc_codes[DN_VLC_N];                // index (level << 1 | run) + 2 * max_level, as ctx->vlc_codes after its offset
    uint8_t vlc_bits[DN_VLC_N];
    uint16_t run_codes[64];
    uint8_t run_bits[64];
    uint8_t dc_codes[16], dc_bits[16];
    uint8_t weight[2][64];                       // luma, chroma (zig-zag order)
    uint8_t zz[64];                              // ff_zigzag_direct, the scan with no IDCT permutation
    uint16_t aan[64];                            // ff_aanscales, for ff_convert_matrix behind ff_fdct_ifast
    int max_level;
};

struct DnRc { int ssd, bits; };                  // RCEntry

// one frame as the kernels see it: what encode_init derives (checked and filled on the host) and the frame's part of the workspace
struct DnFrame {
    const uint8_t *data[3];
    int ls[3];
    const DnTables *tab;
    int cid, width, height, bd, il, nf, first_field, fdct, rd, qmax, mbw, mbh, nmb;
    unsigned frame_bits, frame_size, cu_size;
    FFDnxhdRcState *state;
    uint8_t *out;
    int32_t *out_info;
    int32_t *qmat;                               // [2][qmax + 1][64]: qmatrix_l / qmatrix_c (<< 2 at 8 bit)
    int16_t *coef, *samp, *dcq;                  // per field: nmb x 8 blocks of FDCT output, source samples (RD only), quantised DCs
    DnRc *rc;                                    // per field: [qmax - 1][nmb], qscale 1..qmax - 1
    int32_t *rowbits;                            // per field: [qmax - 1][mbh] bits of a row (fast)
    int32_t *var;                                // per field: nmb variances (fast)
    int32_t *order;                              // per field: macroblocks in radix_sort's order (fast)
    uint8_t *mbq;                                // per field: each macroblock's qscale
    int32_t *mbbits;                             // per field: each macroblock's bits at that qscale
    uint32_t *mboff;                             // per field: each macroblock's bit offset in its slice
    uint32_t *rowbytes, *sliceoff;               // per field: [mbh] slice sizes and offsets
    int32_t *status;                             // per field: 0 coded, EINVAL failed or not reached
};

__device__ __forceinline__ int dn_log2_16(unsigned v)            // av_log2_16bit for the values it is given here (below 1 << 16)
{
#ifdef __CUDA_ARCH__
    return v ? 31 - __clz(v) : 0;
#else
    return v ? 31 - __builtin_clz(v) : 0;
#endif
}

// ---- fetch: dnxhd_get_blocks for block i of a macroblock, as int16 samples -------------------------------------------------------------
// Blocks 0..3 are Y0 Y1 U V of the top 8 lines, 4..7 the same of the bottom 8.  On 1080-line pictures the last row's bottom blocks are
// zero (progressive) or mirrored from 4 lines (interlaced): s0 s1 s2 s3 s3 s2 s1 s0 at 8 bit, s3 s2 s1 s0 s0 s1 s2 s3 at 10 bit.
__device__ inline void dn_fetch_samples(const DnFrame &F, int field, int mby, int mbx, int i, int16_t *s)
{
    const int cur_field = F.first_field ^ field, c = i & 3, plane = c < 2 ? 0 : c - 1;
    const ptrdiff_t ls = (ptrdiff_t)F.ls[plane] << F.il;
    const int bs = F.bd == 8 ? 3 : 4;                                       // block_width_l2: 8 samples of 1 or 2 bytes
    const int x = plane ? mbx << bs : (mbx << (bs + 1)) + (c << bs);
    const uint8_t *ptr = F.data[plane] + (F.il && cur_field ? F.ls[plane] : 0) + (ptrdiff_t)(mby << 4) * ls + x;
    int rows[8] = { 0, 1, 2, 3, 4, 5, 6, 7 };
    if (i >= 4) {
        ptr += 8 * ls;
        if (mby + 1 == F.mbh && F.height == 1080) {
            if (!F.il) {
                for (int k = 0; k < 64; k++) s[k] = 0;
                return;
            }
            for (int r = 0; r < 8; r++) rows[r] = F.bd == 8 ? (r < 4 ? r : 7 - r) : (r < 4 ? 3 - r : r - 4);
        }
    }
    for (int r = 0; r < 8; r++) {
        const uint8_t *src = ptr + rows[r] * ls;
        for (int c = 0; c < 8; c++) s[8 * r + c] = F.bd == 8 ? (int16_t)src[c] : (int16_t)reinterpret_cast<const uint16_t *>(src)[c];
    }
}

// the forward DCT of the samples in place: ff_jpeg_fdct_islow_8 (fdct 0), ff_fdct_ifast (2), ff_faandct (6), ff_jpeg_fdct_islow_10 (bd 10)
template <int FDCT> __device__ inline void dn_fdct8(int16_t *b)
{
    int m[8][8];
    for (int r = 0; r < 8; r++) {
        int in[8];
        for (int k = 0; k < 8; k++) in[k] = b[8 * r + k];
        fdct_row<FDCT>(in, m[r]);
    }
    fdct_cols<FDCT>(m);
    for (int k = 0; k < 64; k++) b[k] = (int16_t)m[k >> 3][k & 7];
}
__device__ inline void dn_fdct(const DnFrame &F, int16_t *b)
{
    if (F.bd == 8) {
        if (F.fdct == 2) dn_fdct8<2>(b);
        else if (F.fdct == 6) dn_fdct8<6>(b);
        else dn_fdct8<0>(b);
        return;
    }
    int in[8], o[8];
    for (int r = 0; r < 8; r++) {
        for (int k = 0; k < 8; k++) in[k] = b[8 * r + k];
        f10_islow_1d(in, o, 1, 12);
        for (int k = 0; k < 8; k++) b[8 * r + k] = (int16_t)o[k];
    }
    for (int c = 0; c < 8; c++) {
        for (int k = 0; k < 8; k++) in[k] = b[8 * k + c];
        f10_islow_1d(in, o, -2, 15);
        for (int k = 0; k < 8; k++) b[8 * k + c] = (int16_t)o[k];
    }
}
// the DC after quantisation: (dc + 4) / 8 through h263_aic at 8 bit, (dc + 2) >> 2 at 10 bit; independent of qscale
__device__ __forceinline__ int16_t dn_dc(const DnFrame &F, int dc) { return (int16_t)(F.bd == 8 ? (dc + 4) / 8 : (dc + 2) >> 2); }

// ---- quantisation of an FDCT block at qscale q; returns last_non_zero --------------------------------------------------------------------
__device__ inline int dn_quantize(const DnFrame &F, int16_t *t, int i, int q)
{
    const int32_t *qmat = F.qmat + ((size_t)((i & 2) ? 1 : 0) * (F.qmax + 1) + q) * 64;
    if (F.bd == 8) {
        int max;
        return mpv_quantize(t, true, 8, qmat, 0, F.tab->zz, max);         // DNxHD leaves m.intra_quant_bias at 0
    }
    t[0] = (int16_t)((t[0] + 2) >> 2);
    int last = 0;
    for (int k = 1; k < 64; k++) {                                          // dnxhd_10bit_dct_quantize:112-120
        const int j = F.tab->zz[k];
        const int sign = t[j] >> 15;
        int level = (t[j] ^ sign) - sign;
        level = (int)((unsigned)level * (unsigned)qmat[j]) >> 18;
        t[j] = (int16_t)((level ^ sign) - sign);
        if (level) last = k;
    }
    return last;
}

// the VLC index of a level, clamped into the table so that a level past +-max_level (where the reference reads outside its tables)
// never reads outside this one
__device__ __forceinline__ int dn_vlc_index(const DnTables &T, int level, int run)
{
    level = min(max(level, -T.max_level), T.max_level - 1);
    return 2 * T.max_level + ((level * 2) | (run ? 1 : 0));
}

// dnxhd_calc_ac_bits (it adds run_bits[0], which is 0: no CID lists a run of 0, and the call refuses one that does)
__device__ inline int dn_ac_bits(const DnTables &T, const int16_t *t, int last)
{
    int bits = 0, lnz = 0;
    for (int k = 1; k <= last; k++) {
        const int level = t[T.zz[k]];
        if (level) {
            const int run = k - lnz - 1;
            bits += T.vlc_bits[dn_vlc_index(T, level, run)] + T.run_bits[run];
            lnz = k;
        }
    }
    return bits;
}

// dnxhd_unquantize_c: the quantised DC stays in place
__device__ inline void dn_unquantize(const DnFrame &F, int16_t *t, int i, int q, int last)
{
    const uint8_t *w = F.tab->weight[(i & 2) ? 1 : 0];
    const int unit = F.bd == 10 ? 8 : 32, rnd = F.bd == 10 ? 8 : 32, sh = F.bd == 10 ? 4 : 6;
    for (int k = 1; k <= last; k++) {
        const int j = F.tab->zz[k];
        int level = t[j];
        if (!level) continue;
        const bool neg = level < 0;
        level = (neg ? 1 - 2 * level : 2 * level + 1) * q * w[k];
        if (w[k] != unit) level += rnd;
        level >>= sh;
        t[j] = (int16_t)(neg ? -level : level);
    }
}

// ctx->m.idsp.idct in place: ff_simple_idct_8 or ff_simple_idct_10
__device__ inline void dn_idct(const DnFrame &F, int16_t *t)
{
    if (F.bd == 8) {
        enc_idct_rows(t);
        int o[8];
        for (int c = 0; c < 8; c++) {
            enc_idct_col(t + c, o);
            for (int k = 0; k < 8; k++) t[8 * k + c] = (int16_t)o[k];
        }
        return;
    }
    uint4 *r = reinterpret_cast<uint4 *>(t);
    for (int k = 0; k < 8; k++) r[k] = i10_row(r[k]);
    for (int c = 0; c < 8; c++) {
        uint32_t w[8];
        for (int k = 0; k < 8; k++) {
            const uint4 v = r[k];
            w[k] = (c >> 1) == 0 ? v.x : (c >> 1) == 1 ? v.y : (c >> 1) == 2 ? v.z : v.w;
        }
        int o[8];
        if (c & 1) i10_col<1>(w, o); else i10_col<0>(w, o);
        for (int k = 0; k < 8; k++) {
            // the column results go back into the packed rows once all columns of this pair are done
            uint4 &v = r[k];
            uint32_t &x = (c >> 1) == 0 ? v.x : (c >> 1) == 1 ? v.y : (c >> 1) == 2 ? v.z : v.w;
            x = (c & 1) ? (x & 0xffffu) | ((uint32_t)(uint16_t)o[k] << 16) : (x & 0xffff0000u) | (uint16_t)o[k];
        }
    }
}

// the DC predictors of a macroblock's blocks: the previous block of the same component in coding order (Y 0 1 4 5, U 2 6, V 3 7), across
// the row; a row starts at 1 << (bit_depth + 2)
__device__ __forceinline__ int dn_comp(int i) { return (i & 2) ? 1 + (i & 1) : 0; }
__device__ inline void dn_row_dc_start(const DnFrame &F, const int16_t *dcq_mb, int mbx, int (&last_dc)[3])
{
    if (!mbx) { last_dc[0] = last_dc[1] = last_dc[2] = 1 << (F.bd + 2); return; }
    last_dc[0] = dcq_mb[-8 + 5]; last_dc[1] = dcq_mb[-8 + 6]; last_dc[2] = dcq_mb[-8 + 7];
}

// dnxhd_calc_bits_thread for one macroblock at qscale q: its bits and, in RD mode, its SSD
__device__ inline DnRc dn_mb_rate(const DnFrame &F, int field, int mb, int q)
{
    const DnTables &T = *F.tab;
    const size_t b0 = ((size_t)field * F.nmb + mb) * 8;
    int last_dc[3];
    dn_row_dc_start(F, F.dcq + b0, mb % F.mbw, last_dc);
    int ac = 0, dcb = 0, ssd = 0;
    alignas(16) int16_t t[64];
    for (int i = 0; i < 8; i++) {
        const int16_t *src = F.coef + (b0 + i) * 64;
        for (int k = 0; k < 64; k++) t[k] = src[k];
        const int last = dn_quantize(F, t, i, q);
        ac += dn_ac_bits(T, t, last);
        const int n = dn_comp(i), diff = t[0] - last_dc[n];
        const int nbits = dn_log2_16(diff < 0 ? -2 * diff : 2 * diff);
        dcb += T.dc_bits[nbits] + nbits;
        last_dc[n] = t[0];
        if (F.rd) {
            dn_unquantize(F, t, i, q, last);
            dn_idct(F, t);
            const int16_t *s = F.samp + (b0 + i) * 64;
            for (int k = 0; k < 64; k++) ssd += (t[k] - s[k]) * (t[k] - s[k]);
        }
    }
    return DnRc{ ssd, ac + dcb + 12 + 8 * T.vlc_bits[2 * T.max_level] };
}

// dnxhd_mb_var_thread for one macroblock (values are never negative: the 8-bit formula by Cauchy-Schwarz, the 10-bit one on truncated means)
__device__ inline int dn_mb_var(const DnFrame &F, int field, int mby, int mbx)
{
    const int cur_field = F.first_field ^ field;
    const ptrdiff_t ls = (ptrdiff_t)F.ls[0] << F.il;
    const uint8_t *base = F.data[0] + (F.il && cur_field ? F.ls[0] : 0) + (ptrdiff_t)(mby << 4) * ls;
    if (F.bd == 8) {
        const uint8_t *pix = base + (mbx << 4);
        const int h = F.height >> F.il;
        const bool partial = mby == F.mbh - 1 && (h & 0xF);
        int bw = 16, bh = 16;
        if (partial || mbx * 16 > F.width - 16) { bw = min(F.width - 16 * mbx, 16); bh = min(h - 16 * mby, 16); }
        int sum = 0, varc = 0;
        for (int y = 0; y < bh; y++)
            for (int x = 0; x < bw; x++) { const int v = pix[x + y * ls]; sum += v; varc += v * v; }
        return (int)(((unsigned)varc - (((unsigned)sum * (unsigned)sum) >> 8) + 128) >> 8);
    }
    const uint8_t *pix = base + (mbx << 5);          // all 16 lines, on 1080-line pictures 8 past the last
    int sum = 0, sqsum = 0;
    for (int y = 0; y < 16; y++)
        for (int x = 0; x < 16; x++) {
            const int v = reinterpret_cast<const uint16_t *>(pix + y * ls)[x] >> 6;
            sum += v; sqsum += v * v;
        }
    const int mean = sum >> 8, sqmean = sqsum >> 8;
    return sqmean - mean * mean;
}

// ---- the coder: put_bits MSB-first into 32-bit big-endian words ORed into a zeroed packet, from any bit offset -----------------------------
__device__ __forceinline__ void dn_or_word(uint32_t *p, uint32_t v)
{
#ifdef AVB_HOSTSIM
    *p |= __builtin_bswap32(v);                      // the host build runs one thread at a time
#else
    atomicOr(p, __byte_perm(v, 0, 0x0123));          // the first and last words are shared with the neighbouring macroblocks
#endif
}
struct DnWriter {
    uint32_t *w;
    unsigned long long acc = 0;
    int n;
    __device__ DnWriter(uint32_t *words, size_t bitpos) : w(words + (bitpos >> 5)), n((int)(bitpos & 31)) {}
    __device__ void put(int bits, uint32_t v)
    {
        if (!bits) return;
        acc = (acc << bits) | v;
        n += bits;
        if (n >= 32) { n -= 32; dn_or_word(w++, (uint32_t)(acc >> n)); }
    }
    __device__ void flush() { if (n) dn_or_word(w, (uint32_t)(acc << (32 - n))); }
};

// dnxhd_encode_thread for one macroblock at its qscale (dnxhd_encode_dc, dnxhd_encode_block), from bit `bitpos` of the coding unit
__device__ inline void dn_write_mb(const DnFrame &F, int field, int mb, uint32_t *cu, size_t bitpos)
{
    const DnTables &T = *F.tab;
    const size_t b0 = ((size_t)field * F.nmb + mb) * 8;
    const int q = F.mbq[(size_t)field * F.nmb + mb];
    int last_dc[3];
    dn_row_dc_start(F, F.dcq + b0, mb % F.mbw, last_dc);
    DnWriter pb(cu, bitpos);
    pb.put(12, (uint32_t)q << 1);
    alignas(16) int16_t t[64];
    for (int i = 0; i < 8; i++) {
        const int16_t *src = F.coef + (b0 + i) * 64;
        for (int k = 0; k < 64; k++) t[k] = src[k];
        const int last = dn_quantize(F, t, i, q);
        const int n = dn_comp(i);
        int diff = t[0] - last_dc[n], nbits;
        if (diff < 0) { nbits = dn_log2_16(-2 * diff); diff--; }
        else nbits = dn_log2_16(2 * diff);
        pb.put(T.dc_bits[nbits] + nbits, ((uint32_t)T.dc_codes[nbits] << nbits) + ((uint32_t)diff & ((1u << nbits) - 1)));
        last_dc[n] = t[0];
        int lnz = 0;
        for (int k = 1; k <= last; k++) {
            const int level = t[T.zz[k]];
            if (level) {
                const int run = k - lnz - 1, idx = dn_vlc_index(T, level, run);
                pb.put(T.vlc_bits[idx], T.vlc_codes[idx]);
                if (run) pb.put(T.run_bits[run], T.run_codes[run]);
                lnz = k;
            }
        }
        pb.put(T.vlc_bits[2 * T.max_level], T.vlc_codes[2 * T.max_level]);      // EOB
    }
    pb.flush();
}

}  // namespace avb
