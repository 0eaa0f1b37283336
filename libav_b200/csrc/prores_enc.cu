// libav_b200/csrc/prores_enc.cu -- the ProRes encoder (libavcodec/proresenc.c: encode_frame with find_quant_thread's rate control) as one
// batched call: n frames to n packets, byte-identical to the reference encoder's for the same frames and options.
//
// The stages, each a kernel whose threads never communicate (so the file also compiles for tests/hostsim/), arithmetic in prores_enc.cuh:
//   1. fetch   one thread per 8 x 8 block: get_slice_data's edge emulation and prores_fdct (the 10-bit islow of fdct10.cuh), staged per
//              plane in macroblock order; one thread per macroblock line of alpha (get_alpha_data).
//   2. estimate one thread per (slice, trellis node): the bits and error of min_quant..max_quant, and for the last node the search past
//              max_quant (q up to 127, 128 when nothing fits, quant_mat * q throughout).
//   3. trellis one thread per macroblock row of a picture: find_slice_quant's trellis (:866-901) and find_quant_thread's backtrack.
//   4. sizes   one thread per (slice, plane): the exact bytes of the plane at its quantiser, counted by the coder itself (the alpha estimate
//              is not a size: it counts a run as 4 / 15 bits where put_alpha_run writes 5 / 16, and is not rounded to bytes).
//   5. layout  one thread per frame: slice offsets, picture and frame sizes, and the capacity check.
//   6. write   one thread per (slice, plane): the plane's bits, and the headers and seek tables around them.
// Under force_quant stages 2 and 3 are skipped: every slice takes the forced quantiser.
#include "common.cuh"
#include "prores_enc.cuh"
#include "../../include/avdsp_b200.h"
#include <string.h>

namespace avb {
namespace {

constexpr int PE_FRAMES_PER_LAUNCH = 8;
struct PeLaunch { PeFrame f[PE_FRAMES_PER_LAUNCH]; };

// proresenc.c's tables, restated: the quantiser matrices, per profile min_quant, max_quant, br_tab and the matrix, and prores_mb_limits
const uint8_t pe_quant_matrices[5][64] = {
    { 4,  7,  9, 11, 13, 14, 15, 63,  7,  7, 11, 12, 14, 15, 63, 63,  9, 11, 13, 14, 15, 63, 63, 63, 11, 11, 13, 14, 63, 63, 63, 63,
     11, 13, 14, 63, 63, 63, 63, 63, 13, 14, 63, 63, 63, 63, 63, 63, 13, 63, 63, 63, 63, 63, 63, 63, 63, 63, 63, 63, 63, 63, 63, 63 },
    { 4,  5,  6,  7,  9, 11, 13, 15,  5,  5,  7,  8, 11, 13, 15, 17,  6,  7,  9, 11, 13, 15, 15, 17,  7,  7,  9, 11, 13, 15, 17, 19,
      7,  9, 11, 13, 14, 16, 19, 23,  9, 11, 13, 14, 16, 19, 23, 29,  9, 11, 13, 15, 17, 21, 28, 35, 11, 13, 16, 17, 21, 28, 35, 41 },
    { 4,  4,  5,  5,  6,  7,  7,  9,  4,  4,  5,  6,  7,  7,  9,  9,  5,  5,  6,  7,  7,  9,  9, 10,  5,  5,  6,  7,  7,  9,  9, 10,
      5,  6,  7,  7,  8,  9, 10, 12,  6,  7,  7,  8,  9, 10, 12, 15,  6,  7,  7,  9, 10, 11, 14, 17,  7,  7,  9, 10, 11, 14, 17, 21 },
    { 4,  4,  4,  4,  4,  4,  4,  4,  4,  4,  4,  4,  4,  4,  4,  4,  4,  4,  4,  4,  4,  4,  4,  4,  4,  4,  4,  4,  4,  4,  4,  5,
      4,  4,  4,  4,  4,  4,  5,  5,  4,  4,  4,  4,  4,  5,  5,  6,  4,  4,  4,  4,  5,  5,  6,  7,  4,  4,  4,  4,  5,  6,  7,  7 },
    { 4,  4,  4,  4,  4,  4,  4,  4,  4,  4,  4,  4,  4,  4,  4,  4,  4,  4,  4,  4,  4,  4,  4,  4,  4,  4,  4,  4,  4,  4,  4,  4,
      4,  4,  4,  4,  4,  4,  4,  4,  4,  4,  4,  4,  4,  4,  4,  4,  4,  4,  4,  4,  4,  4,  4,  4,  4,  4,  4,  4,  4,  4,  4,  4 },
};
struct PeProfile { int min_quant, max_quant, br_tab[4], quant; };
const PeProfile pe_profiles[5] = {
    { 4, 8, { 300, 242, 220, 194 }, 0 },           // proxy
    { 1, 9, { 720, 560, 490, 440 }, 1 },           // LT
    { 1, 6, { 1050, 808, 710, 632 }, 2 },          // standard
    { 1, 6, { 1566, 1216, 1070, 950 }, 3 },        // high quality
    { 1, 6, { 2350, 1828, 1600, 1425 }, 3 },       // 4444
};
const int pe_mb_limits[4] = { 1620, 2700, 6075, 9216 };

// ---- kernels ------------------------------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(128) pe_fetch_kernel(const __grid_constant__ PeLaunch L)
{
    const PeFrame &F = L.f[blockIdx.y];
    // 32-bit indices: a frame holds at most 4096 x 4096 macroblocks of 12 blocks
    const unsigned ncb = F.c444 ? 4 : 2, bpm = 4 + 2 * ncb;
    const unsigned mbs_pic = (unsigned)F.mbw * F.mbh, per_pic = mbs_pic * bpm;
    const unsigned i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= per_pic * F.ppf) return;
    const int pic = i >= per_pic;
    unsigned r = i - pic * per_pic, m;
    int p, b;
    if (r < mbs_pic * 4) { p = 0; m = r >> 2; b = (int)(r & 3); }
    else {
        r -= mbs_pic * 4;
        p = r < mbs_pic * ncb ? 1 : 2;
        r -= (p - 1) * mbs_pic * ncb;
        m = r / ncb; b = (int)(r % ncb);
    }
    pe_fetch_fdct(F, pic, p, (int)(m / F.mbw), (int)(m % F.mbw), b, F.coef + 64 * (size_t)i);
}

// one line of one macroblock of alpha, into its slice's 16 x (16 * mbs) raster
__global__ void __launch_bounds__(128) pe_alpha_kernel(const __grid_constant__ PeLaunch L)
{
    const PeFrame &F = L.f[blockIdx.y];
    const unsigned mbs_pic = (unsigned)F.mbw * F.mbh;
    const unsigned i = blockIdx.x * blockDim.x + threadIdx.x;
    if (!F.abits || i >= mbs_pic * F.ppf * 16) return;
    const int line = (int)(i & 15);
    const unsigned mb = i >> 4;
    const int pic = mb >= mbs_pic, mby = (int)((mb - pic * mbs_pic) / F.mbw), mbx = (int)(mb % F.mbw);
    int x0, mbs;
    pe_slice_of_mb(F, mbx, x0, mbs);
    int16_t *dst = F.alpha + ((size_t)pic * mbs_pic + (size_t)mby * F.mbw + x0) * 256 + line * 16 * mbs + (mbx - x0) * 16;
    pe_fetch_alpha(F, pic, mby, mbx, line, dst);
}

// find_slice_quant:806-864 for node k of slice s: k < nq - 1 is q = min_quant + k; the last node is the overquant one
__global__ void __launch_bounds__(128, 4) pe_estimate_kernel(const __grid_constant__ PeLaunch L)
{
    const PeFrame &F = L.f[blockIdx.y];
    const unsigned i = blockIdx.x * blockDim.x + threadIdx.x;
    if (F.force_quant || i >= (unsigned)F.nslices * F.nq) return;
    const int s = (int)(i / F.nq), k = (int)(i % F.nq);
    const int pic = s / F.spp, row = (s % F.spp) / F.sw, col = s % F.sw;
    const PeSlice S = pe_slice(F, pic, row, col);
    PeEst &E = F.est[s];
    const int limit = F.bits_per_mb * S.mbs;
    // one estimate per pass: node k's quantiser, or for the last node max_quant and then, while the slice does not fit, every q past it
    int q = k < F.nq - 1 ? F.minq + k : F.maxq;
    for (;;) {
        int error;
        const int bits = pe_est_slice(F, S, q, error);
        if (q <= F.maxq && bits > 65000 * 8) error = PE_SCORE_LIMIT;     // the past-max_quant search has no such cap
        if (k < F.nq - 1) { E.bits[k] = bits; E.score[k] = error; return; }
        if (q == F.maxq && bits <= limit) { E.bits[k] = bits; E.score[k] = error + 1; E.overquant = q; return; }
        if (q > F.maxq && (bits <= limit || q == 127)) {                 // nothing fits: the search ends at 128 with q = 127's estimate
            E.bits[k] = bits; E.score[k] = error; E.overquant = bits <= limit ? q : 128;
            return;
        }
        q++;
    }
}

// find_slice_quant:866-901 over a macroblock row, then find_quant_thread's backtrack into the slices' quantisers
__global__ void __launch_bounds__(128) pe_trellis_kernel(const __grid_constant__ PeLaunch L)
{
    const PeFrame &F = L.f[blockIdx.y];
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= F.ppf * F.mbh) return;
    const int s0 = (i / F.mbh) * F.spp + (i % F.mbh) * F.sw;
    if (F.force_quant) {
        for (int c = 0; c < F.sw; c++) F.sq[s0 + c] = F.force_quant;
        return;
    }
    const int nq = F.nq;
    int pbits[PE_NQ], pscore[PE_NQ], cbits[PE_NQ], cscore[PE_NQ];
    for (int k = 0; k < PE_NQ; k++) { pbits[k] = 0; pscore[k] = 0; }
    int mbs_done = 0;
    for (int c = 0; c < F.sw; c++) {
        int x0, mbs;
        pe_slice_span(F, c, x0, mbs);
        mbs_done += mbs;
        const PeEst &E = F.est[s0 + c];
        const int bits_limit = mbs_done * F.bits_per_mb;
        int8_t *back = F.back + (size_t)(s0 + c) * PE_NQ;
        for (int q = 0; q < nq; q++) back[q] = -1;
        for (int pq = 0; pq < nq; pq++) {
            for (int q = 0; q < nq; q++) {
                const int bits = pbits[pq] + E.bits[q];
                int error = E.score[q];
                if (bits > bits_limit) error = PE_SCORE_LIMIT;
                const int new_score = pscore[pq] < PE_SCORE_LIMIT && error < PE_SCORE_LIMIT ? pscore[pq] + error : PE_SCORE_LIMIT;
                if (back[q] == -1 || cscore[q] >= new_score) {        // equal scores: the later pq wins
                    cbits[q] = bits; cscore[q] = new_score; back[q] = (int8_t)pq;
                }
            }
        }
        for (int q = 0; q < nq; q++) { pbits[q] = cbits[q]; pscore[q] = cscore[q]; }
    }
    int best = 0, error = pscore[0];
    for (int q = 1; q < nq; q++)
        if (pscore[q] <= error) { error = pscore[q]; best = q; }     // equal scores: the later q wins
    for (int c = F.sw - 1; c >= 0; c--) {
        const int s = s0 + c;
        F.sq[s] = best == nq - 1 ? F.est[s].overquant : F.minq + best;
        best = F.back[(size_t)s * PE_NQ + best];
    }
}

__global__ void __launch_bounds__(128) pe_size_kernel(const __grid_constant__ PeLaunch L)
{
    const PeFrame &F = L.f[blockIdx.y];
    const unsigned i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= (unsigned)F.nslices * 4) return;
    const int s = (int)(i >> 2), p = (int)(i & 3);
    if (p == 3 && !F.abits) { F.size[i] = 0; return; }
    const PeSlice S = pe_slice(F, s / F.spp, (s % F.spp) / F.sw, s % F.sw);
    PeCount c;
    pe_code_slice_plane(c, F, S, p, F.sq[s]);
    F.size[i] = (uint32_t)((c.bits + 7) >> 3);
}

__device__ inline int pe_frame_header_size(const PeFrame &F) { return 20 + (F.matrix ? 128 : 0); }
__device__ inline int pe_slice_header_size(const PeFrame &F) { return F.abits ? 8 : 6; }

__global__ void __launch_bounds__(32) pe_layout_kernel(const __grid_constant__ PeLaunch L)
{
    const PeFrame &F = L.f[blockIdx.y];
    if (threadIdx.x) return;
    const int hs = pe_slice_header_size(F);
    size_t pos = 8 + pe_frame_header_size(F);
    for (int pic = 0; pic < F.ppf; pic++) {
        const size_t start = pos;
        pos += 8 + 2 * (size_t)F.spp;
        for (int k = 0; k < F.spp; k++) {
            const int s = pic * F.spp + k;
            F.off[s] = (uint32_t)pos;
            const uint32_t *z = F.size + 4 * (size_t)s;
            pos += hs + z[0] + z[1] + z[2] + z[3];
        }
        F.pic_size[pic] = (uint32_t)(pos - start);
    }
    *F.out_size = pos <= F.cap ? (int32_t)pos : -(int32_t)pos;
}

__device__ inline void pe_be16(uint8_t *p, unsigned v) { p[0] = (uint8_t)(v >> 8); p[1] = (uint8_t)v; }
__device__ inline void pe_be32(uint8_t *p, unsigned v) { pe_be16(p, v >> 16); pe_be16(p + 2, v); }

__global__ void __launch_bounds__(128) pe_write_kernel(const __grid_constant__ PeLaunch L)
{
    const PeFrame &F = L.f[blockIdx.y];
    const unsigned i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= (unsigned)F.nslices * 4 || *F.out_size <= 0) return;
    const int s = (int)(i >> 2), p = (int)(i & 3);
    if (p == 3 && !F.abits) return;
    const int pic = s / F.spp, k = s % F.spp, hs = pe_slice_header_size(F);
    const uint32_t *z = F.size + 4 * (size_t)s;
    uint8_t *slice = F.out + F.off[s];
    // the planes follow the header in order: luma, chroma, chroma, alpha
    size_t at = hs;
    for (int j = 0; j < p; j++) at += z[j];
    const PeSlice S = pe_slice(F, pic, k / F.sw, k % F.sw);
    PeWriter w(slice + at);
    pe_code_slice_plane(w, F, S, p, F.sq[s]);
    w.flush();
    if (p) return;
    // slice header: its size in bits, the quantiser, the size of every plane but the last; the seek table's entry
    const int np = F.abits ? 4 : 3;
    uint32_t total = hs;
    slice[0] = (uint8_t)(hs << 3);
    slice[1] = (uint8_t)F.sq[s];
    for (int j = 0; j < np - 1; j++) pe_be16(slice + 2 + 2 * j, z[j]);
    for (int j = 0; j < np; j++) total += z[j];
    const size_t pic_start = F.off[pic * F.spp] - 8 - 2 * (size_t)F.spp;
    pe_be16(F.out + pic_start + 8 + 2 * k, total);
    if (k) return;
    // picture header; progressive pictures store 7 bytes less than their size (buf - picture_size_pos - 6)
    uint8_t *ph = F.out + pic_start;
    ph[0] = 0x40;
    pe_be32(ph + 1, F.ppf == 1 ? F.pic_size[pic] - 7 : F.pic_size[pic]);
    pe_be16(ph + 5, F.spp);
    ph[7] = (uint8_t)(F.lmps << 4);
    if (pic) return;
    // frame atom and frame header
    uint8_t *o = F.out;
    const int fh = pe_frame_header_size(F);
    pe_be32(o, (unsigned)*F.out_size);
    o[4] = 'i'; o[5] = 'c'; o[6] = 'p'; o[7] = 'f';
    pe_be16(o + 8, fh);
    pe_be16(o + 10, 0);
    for (int j = 0; j < 4; j++) o[12 + j] = F.vendor[j];
    pe_be16(o + 16, F.width);
    pe_be16(o + 18, F.height);
    o[20] = (uint8_t)(((F.c444 ? 3 : 2) << 6) | (F.ppf == 1 ? 0 : F.tff ? 0x04 : 0x08));
    o[21] = 0;
    o[22] = F.prim; o[23] = F.trc; o[24] = F.csp;
    o[25] = (uint8_t)(0x40 | (F.abits >> 3));
    o[26] = 0;
    o[27] = F.matrix ? 0x03 : 0x00;
    if (F.matrix)                                             // the one matrix twice: luma, then chroma
        for (int j = 0; j < 128; j++) o[28 + j] = F.qm[j & 63];
}

// ---- host side ------------------------------------------------------------------------------------------------------------------------------
int pe_refuse(const char *msg) { set_error_msg("ff_prores_encode_frames_cuda", msg); return -1; }

size_t pe_align(size_t v) { return (v + 255) & ~(size_t)255; }

// encode_init's checks and derivations for one frame; the frame's workspace bytes.  Fills F's geometry (not its workspace pointers).
int pe_frame(const FFProresEncodeWork &w, PeFrame &F, size_t &bytes)
{
    if (w.pix_fmt < 0 || w.pix_fmt > 2) return pe_refuse("pix_fmt must be 0 (yuv422p10), 1 (yuv444p10) or 2 (yuva444p10)");
    if (w.interlaced < 0 || w.interlaced > 2) return pe_refuse("interlaced must be 0, 1 (top field first) or 2 (bottom field first)");
    if (w.profile < 0 || w.profile > 4) return pe_refuse("profile must be 0..4");
    if (w.mbs_per_slice != 1 && w.mbs_per_slice != 2 && w.mbs_per_slice != 4 && w.mbs_per_slice != 8)
        return pe_refuse("mbs_per_slice must be 1, 2, 4 or 8");
    if (w.quant_sel < -1 || w.quant_sel > 4) return pe_refuse("quant_sel must be -1..4");
    if (w.force_quant < 0 || w.force_quant > 64) return pe_refuse("force_quant must be 0..64");
    if (w.bits_per_mb < 0 || w.bits_per_mb > 8192 || (!w.force_quant && w.bits_per_mb > 0 && w.bits_per_mb < 128))
        return pe_refuse("bits_per_mb must be 0 or 128..8192");
    const bool has_alpha = w.pix_fmt == 2;
    if (has_alpha && w.alpha_bits != 0 && w.alpha_bits != 8 && w.alpha_bits != 16) return pe_refuse("alpha_bits must be 0, 8 or 16");
    for (int j = 0; j < 4; j++)
        if (!w.vendor[j]) return pe_refuse("the vendor ID must be 4 non-zero bytes");
    if (w.width < 1 || w.height < 1 || w.width > 65535 || w.height > 65535) return pe_refuse("width and height must be 1..65535");
    memset(&F, 0, sizeof(F));
    F.width = w.width; F.height = w.height; F.c444 = w.pix_fmt != 0; F.abits = has_alpha ? w.alpha_bits : 0;
    F.ppf = w.interlaced ? 2 : 1; F.tff = w.interlaced == 1;
    const int np = F.abits ? 4 : 3;
    for (int p = 0; p < np; p++) {
        if (!w.data[p] || ((uintptr_t)w.data[p] & 1)) return pe_refuse("NULL or odd plane pointer");
        if (w.linesize[p] <= 0 || (w.linesize[p] & 1)) return pe_refuse("linesize must be even and positive");
        const long pw = (p == 1 || p == 2) && !F.c444 ? (w.width + 1) >> 1 : w.width;
        if (w.linesize[p] < 2 * pw) return pe_refuse("linesize narrower than the plane");
        F.data[p] = w.data[p]; F.ls[p] = w.linesize[p];
    }
    F.mbw = (w.width + 15) >> 4;
    F.mbh = w.interlaced ? (w.height + 31) >> 5 : (w.height + 15) >> 4;
    if (w.interlaced && w.height / 2 <= 16 * (F.mbh - 1))
        return pe_refuse("interlaced height leaves a field's last macroblock row without lines (height 1 or 32k + 1)");
    F.mps = w.mbs_per_slice;
    F.lmps = F.mps == 1 ? 0 : F.mps == 2 ? 1 : F.mps == 4 ? 2 : 3;
    const int rest = F.mbw - (F.mbw / F.mps) * F.mps;
    F.sw = F.mbw / F.mps + (rest & 1) + ((rest >> 1) & 1) + ((rest >> 2) & 1);
    if ((long)F.sw * F.mbh > 65535) return pe_refuse("more than 65535 slices per picture");
    F.spp = F.sw * F.mbh; F.nslices = F.spp * F.ppf;
    if (!w.out || !w.out_size || ((uintptr_t)w.out_size & 3)) return pe_refuse("NULL packet buffer, or a NULL or misaligned out_size");
    const PeProfile &P = pe_profiles[w.profile];
    const int qsel = w.quant_sel == -1 ? P.quant : w.quant_sel;
    memcpy(F.qm, pe_quant_matrices[qsel], 64);
    F.matrix = qsel != 4;
    F.scan = w.interlaced ? 1 : 0;
    F.force_quant = w.force_quant;
    F.minq = P.min_quant; F.maxq = P.max_quant; F.nq = P.max_quant - P.min_quant + 2;
    F.bits_per_mb = w.bits_per_mb;
    if (!F.force_quant && !F.bits_per_mb) {
        int i;
        for (i = 0; i < 3; i++)
            if (pe_mb_limits[i] >= F.mbw * F.mbh * F.ppf) break;
        F.bits_per_mb = P.br_tab[i];
    }
    memcpy(F.vendor, w.vendor, 4);
    F.prim = w.color_primaries; F.trc = w.color_trc; F.csp = w.colorspace;
    F.out = w.out; F.cap = w.out_capacity; F.out_size = w.out_size;
    const size_t mbs = (size_t)F.mbw * F.mbh * F.ppf;
    bytes = pe_align(mbs * (4 + 2 * (F.c444 ? 4 : 2)) * 128) + (F.abits ? pe_align(mbs * 512) : 0) +
            pe_align((size_t)F.nslices * sizeof(PeEst)) + pe_align((size_t)F.nslices * PE_NQ) + pe_align((size_t)F.nslices * 4) +
            pe_align((size_t)F.nslices * 16) + pe_align((size_t)F.nslices * 4) + 256;
    return 0;
}

void pe_place(PeFrame &F, uint8_t *&ws)
{
    const size_t mbs = (size_t)F.mbw * F.mbh * F.ppf;
    F.coef = reinterpret_cast<int16_t *>(ws); ws += pe_align(mbs * (4 + 2 * (F.c444 ? 4 : 2)) * 128);
    F.alpha = nullptr;
    if (F.abits) { F.alpha = reinterpret_cast<int16_t *>(ws); ws += pe_align(mbs * 512); }
    F.est = reinterpret_cast<PeEst *>(ws); ws += pe_align((size_t)F.nslices * sizeof(PeEst));
    F.back = reinterpret_cast<int8_t *>(ws); ws += pe_align((size_t)F.nslices * PE_NQ);
    F.sq = reinterpret_cast<int32_t *>(ws); ws += pe_align((size_t)F.nslices * 4);
    F.size = reinterpret_cast<uint32_t *>(ws); ws += pe_align((size_t)F.nslices * 16);
    F.off = reinterpret_cast<uint32_t *>(ws); ws += pe_align((size_t)F.nslices * 4);
    F.pic_size = reinterpret_cast<uint32_t *>(ws); ws += 256;
}

size_t pe_workspace(const FFProresEncodeWork *frames, int n)
{
    if (!frames || n < 1) return 0;
    size_t total = 0;
    for (int k = 0; k < n; k++) {
        PeFrame F;
        size_t b;
        if (pe_frame(frames[k], F, b)) return 0;
        total += b;
    }
    return total;
}

unsigned pe_blocks(size_t threads) { return (unsigned)((threads + 127) / 128); }
size_t pe_max(size_t a, size_t b) { return a > b ? a : b; }

int pe_launch(PeLaunch &L, int m, cudaStream_t st)
{
    size_t nblk = 0, nalpha = 0, nest = 0, nrows = 0, nplanes = 0;
    for (int k = 0; k < m; k++) {
        const PeFrame &F = L.f[k];
        const size_t mbs = (size_t)F.mbw * F.mbh * F.ppf;
        nblk = pe_max(nblk, mbs * (4 + 2 * (F.c444 ? 4 : 2)));
        nalpha = pe_max(nalpha, F.abits ? mbs * 16 : 0);
        nest = pe_max(nest, F.force_quant ? 0 : (size_t)F.nslices * F.nq);
        nrows = pe_max(nrows, (size_t)F.ppf * F.mbh);
        nplanes = pe_max(nplanes, (size_t)F.nslices * 4);
    }
    const char *where = "ff_prores_encode_frames_cuda";
    AVB_LAUNCH(pe_fetch_kernel, dim3(pe_blocks(nblk), m), dim3(128), 0, st)(L);
    if (check_launch(where)) return -1;
    if (nalpha) {
        AVB_LAUNCH(pe_alpha_kernel, dim3(pe_blocks(nalpha), m), dim3(128), 0, st)(L);
        if (check_launch(where)) return -1;
    }
    if (nest) {
        AVB_LAUNCH(pe_estimate_kernel, dim3(pe_blocks(nest), m), dim3(128), 0, st)(L);
        if (check_launch(where)) return -1;
    }
    AVB_LAUNCH(pe_trellis_kernel, dim3(pe_blocks(nrows), m), dim3(128), 0, st)(L);
    if (check_launch(where)) return -1;
    AVB_LAUNCH(pe_size_kernel, dim3(pe_blocks(nplanes), m), dim3(128), 0, st)(L);
    if (check_launch(where)) return -1;
    AVB_LAUNCH(pe_layout_kernel, dim3(1, m), dim3(32), 0, st)(L);
    if (check_launch(where)) return -1;
    AVB_LAUNCH(pe_write_kernel, dim3(pe_blocks(nplanes), m), dim3(128), 0, st)(L);
    return check_launch(where);
}

}  // namespace
}  // namespace avb

using namespace avb;

extern "C" {

size_t ff_prores_encode_workspace_cuda(const FFProresEncodeWork *frames, int n)
{
    return pe_workspace(frames, n);
}

int ff_prores_encode_frames_cuda(const FFProresEncodeWork *frames, int n, void *workspace, size_t workspace_bytes, void *stream)
{
    avb::enter();
    if (n == 0) return 0;
    if (!frames || n < 0) return pe_refuse("NULL frames or a negative count");
    size_t need = 0;
    for (int k = 0; k < n; k++) {                         // every frame is checked before anything is launched
        PeFrame F;
        size_t b;
        if (pe_frame(frames[k], F, b)) return -1;
        need += b;
    }
    if (!workspace || workspace_bytes < need) return pe_refuse("workspace missing or smaller than ff_prores_encode_workspace_cuda returns");
    uint8_t *ws = (uint8_t *)workspace;
    for (int g0 = 0; g0 < n; g0 += PE_FRAMES_PER_LAUNCH) {
        const int m = n - g0 < PE_FRAMES_PER_LAUNCH ? n - g0 : PE_FRAMES_PER_LAUNCH;
        PeLaunch L;
        memset(&L, 0, sizeof(L));
        for (int k = 0; k < m; k++) {
            size_t b;
            pe_frame(frames[g0 + k], L.f[k], b);
            pe_place(L.f[k], ws);
        }
        if (pe_launch(L, m, (cudaStream_t)stream)) return -1;
    }
    return 0;
}

}  // extern "C"
