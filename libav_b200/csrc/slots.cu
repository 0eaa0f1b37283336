// libav_b200/csrc/slots.cu -- per-call slot functions and the ff_*_init_cuda hooks for FDCTDSPContext, MECmpContext,
// H264DSPContext, H264QpelContext, H264ChromaContext and HpelDSPContext (IDCTDSP / BlockDSP live in capi_idct.cu).
//
// A slot has the C slot's exact signature and HOST pointers.  It stages the rectangles the C function would touch
// into one pinned buffer (compact pitch), uploads it, runs the same device arithmetic as the batched kernels (a batch
// of one), downloads and scatters the rectangles the C function may modify, and synchronises.  This is the drop-in /
// parity path behind the reference's arch dispatch; throughput comes from the batched entry points.
#include "h264dsp.cuh"
#include "scratch.h"
#include "../../include/avdsp_b200.h"
#include <string.h>

namespace avb {

constexpr int SP = 32;            // pitch of every staged pixel rectangle
enum SlotOp {
    OP_H264_IDCT, OP_H264_IDCT_MB, OP_H264_LUMA_DC, OP_H264_CHROMA_DC, OP_H264_ADD_PIXELS, OP_H264_LOOP, OP_H264_QPEL, OP_H264_CHROMA_MC,
};
struct SlotArgs {
    int op, a, b, c, d, e, f;                 // op-specific integers
    uint8_t *p0, *p1, *p2;                    // device rectangles / buffers
    int16_t *blk;                             // device coefficient buffer
    int off[48];                              // block offsets (idct_mb)
    uint8_t nnzc[120];
    int8_t tc0[4];
};

struct DirectFetch {
    const uint8_t *p; int stride;
    __device__ __forceinline__ int operator()(int x, int y) const { return p[y * stride + x]; }
};

__global__ void __launch_bounds__(32) slot_kernel(SlotArgs s)
{
    const int lane = threadIdx.x;
    switch (s.op) {
    case OP_H264_IDCT:                        // a = which (0 idct4, 1 idct8, 2 dc4, 3 dc8)
        if (lane == 0) {
            if (s.a == 0) h264_idct4_add(s.p0, s.blk, SP);
            else if (s.a == 1) h264_idct8_add(s.p0, s.blk, SP);
            else h264_dc_add(s.p0, s.blk, SP, s.a == 2 ? 4 : 8);
        }
        break;
    case OP_H264_IDCT_MB: {                   // a = which (0 add16, 1 add16intra, 2 idct8_add4, 3 add8, 4 add8_422), b = pitch
        const int which = s.a, pitch = s.b;
        if (which < 3 && lane < 16) {
            int16_t *blk = s.blk + 16 * lane;
            uint8_t *d = s.p0 + s.off[lane];
            const int nnz = s.nnzc[scan8_of(lane)];
            if (which == 0) { if (nnz) { if (nnz == 1 && blk[0]) h264_dc_add(d, blk, pitch, 4); else h264_idct4_add(d, blk, pitch); } }
            else if (which == 1) { if (nnz) h264_idct4_add(d, blk, pitch); else if (blk[0]) h264_dc_add(d, blk, pitch, 4); }
            else if ((lane & 3) == 0 && nnz) { if (nnz == 1 && blk[0]) h264_dc_add(d, blk, pitch, 8); else h264_idct8_add(d, blk, pitch); }
        } else if (which >= 3 && lane < (which == 4 ? 16 : 8)) {
            // 4:2:0: four blocks per plane.  4:2:2 (h264idct_template.c:216-236): eight, the lower four keep their coefficients at
            // block i but are addressed through scan8[i + 4] / block_offset[i + 4]
            const int per = which == 4 ? 8 : 4, plane = lane / per, k = lane % per;
            const int i = 16 + 16 * plane + k, e = k >= 4 ? i + 4 : i;
            int16_t *blk = s.blk + 16 * i;
            uint8_t *d = (plane ? s.p1 : s.p0) + s.off[e];
            if (s.nnzc[scan8_of(e)]) h264_idct4_add(d, blk, pitch); else if (blk[0]) h264_dc_add(d, blk, pitch, 4);
        }
    } break;
    case OP_H264_LUMA_DC: if (lane == 0) h264_luma_dc_dequant(s.blk, s.blk + 256, s.a); break;
    case OP_H264_CHROMA_DC: if (lane == 0) { if (s.b) h264_chroma422_dc_dequant(s.blk, s.a); else h264_chroma_dc_dequant(s.blk, s.a); } break;    // b = 4:2:2
    case OP_H264_ADD_PIXELS: {                // a = n (4 / 8): dst += block (wraps, no clip), block cleared
        const int n = s.a;
        for (int i = lane; i < n * n; i += 32) { uint8_t *d = s.p0 + (i / n) * SP + i % n; *d = (uint8_t)(*d + s.blk[i]); s.blk[i] = 0; }
    } break;
    case OP_H264_LOOP: {                      // a = kind bits (1 horizontal edge, 2 chroma, 4 intra), b = alpha, c = beta, d = lines; p0 -> q0 sample
        const bool horiz_edge = s.a & 1, chroma = s.a & 2, intra = s.a & 4;
        const int across = horiz_edge ? SP : 1, along = horiz_edge ? 1 : SP, lines = s.d;      // a tc0 entry covers lines / 4 of them
        if (lane < lines) {
            uint8_t *q = s.p0 + lane * along;
            const int tc = s.tc0[lane / (lines >> 2)];
            if (!chroma) { if (intra) h264_luma_intra_line(q, across, s.b, s.c); else if (tc >= 0) h264_luma_line(q, across, s.b, s.c, tc); }
            else if (intra || tc > 0) h264_chroma_line(q, across, s.b, s.c, tc, intra);
        }
    } break;
    case OP_H264_QPEL: {                      // a = avg, b = size, c = mc; p0 = dst, p1 = src (both pitch SP)
        const DirectFetch S = { s.p1, SP };
        for (int i = lane; i < s.b * s.b; i += 32) {
            const int x = i % s.b, y = i / s.b, v = qpel_sample(S, x, y, s.c & 3, s.c >> 2);
            uint8_t *d = s.p0 + y * SP + x;
            *d = (uint8_t)(s.a ? (*d + v + 1) >> 1 : v);
        }
    } break;
    case OP_H264_CHROMA_MC: {                 // a = avg, b = w, c = h, d = x, e = y
        const DirectFetch S = { s.p1, SP };
        for (int i = lane; i < s.b * s.c; i += 32) {
            const int x = i % s.b, y = i / s.b, v = chroma_sample(S, x, y, s.d, s.e);
            uint8_t *d = s.p0 + y * SP + x;
            *d = (uint8_t)(s.a ? (*d + v + 1) >> 1 : v);
        }
    } break;
    }
}

// ---- staging ------------------------------------------------------------------------------------------
struct Stage {
    ScratchLock lk;
    uint8_t *h = nullptr, *d = nullptr;
    cudaStream_t s = nullptr;
    size_t used = 0;
    static constexpr size_t CAP = 64 * 1024;
    bool ok() {
        Scratch &S = scratch();
        h = (uint8_t *)S.pinned2(CAP); d = (uint8_t *)S.dev(4, CAP);
        cudaStream_t *st = S.streams();
        if (!h || !d || !st) return false;
        s = st[0];
        return true;
    }
    // reserve `bytes` (16-byte aligned); returns the offset
    size_t take(size_t bytes) { size_t o = used; used += (bytes + 15) & ~(size_t)15; return o; }
    size_t rect_in(const uint8_t *src, ptrdiff_t stride, int w, int hgt) {           // rows -> pitch SP
        size_t o = take((size_t)SP * hgt + SP);
        for (int y = 0; y < hgt; y++) memcpy(h + o + (size_t)y * SP, src + y * stride, w);
        return o;
    }
    void rect_out(uint8_t *dst, ptrdiff_t stride, int w, int hgt, size_t o) { for (int y = 0; y < hgt; y++) memcpy(dst + y * stride, h + o + (size_t)y * SP, w); }
    int up() { AVB_CUDA(cudaMemcpyAsync(d, h, used, cudaMemcpyHostToDevice, s), "slot:h2d"); return 0; }
    int down() {
        AVB_CUDA(cudaMemcpyAsync(h, d, used, cudaMemcpyDeviceToHost, s), "slot:d2h");
        AVB_CUDA(cudaStreamSynchronize(s), "slot:sync");
        return 0;
    }
    int run(const SlotArgs &a) { AVB_LAUNCH(slot_kernel, 1, 32, 0, s)(a); return check_launch("slot"); }
};

// H264DSPContext.startcode_find_candidate = ff_startcode_find_candidate_c (libavcodec/startcode.c:31-59): index of the first zero byte, `size`
// when there is none before it.  Thread per byte, the smallest index wins through atomicMin.
__global__ void __launch_bounds__(256) startcode_kernel(const uint8_t *__restrict__ buf, int size, int *__restrict__ first)
{
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < size && !buf[i]) atomicMin(first, i);
}
int startcode_find_candidate_cuda(const uint8_t *buf, int size)
{
    if (size <= 0) return 0;
    ScratchLock lk;
    Scratch &S = scratch();
    const size_t need = (size_t)size + 64;
    uint8_t *h = (uint8_t *)S.pinned2(need), *d = (uint8_t *)S.dev(4, need);
    cudaStream_t *st = S.streams();
    if (!h || !d || !st) return size;
    const size_t off = ((size_t)size + 15) & ~(size_t)15;            // the result word sits after the bytes
    memcpy(h, buf, size);
    memcpy(h + off, &size, 4);
    if (cudaMemcpyAsync(d, h, off + 4, cudaMemcpyHostToDevice, st[0]) != cudaSuccess) { set_error("startcode slot:h2d", cudaGetLastError()); return size; }
    AVB_LAUNCH(startcode_kernel, dim3((unsigned)((size + 255) / 256)), dim3(256), 0, st[0])(d, size, (int *)(d + off));
    if (check_launch("startcode slot")) return size;
    int r = size;
    if (cudaMemcpyAsync(h + off, d + off, 4, cudaMemcpyDeviceToHost, st[0]) != cudaSuccess || cudaStreamSynchronize(st[0]) != cudaSuccess) { set_error("startcode slot:d2h", cudaGetLastError()); return size; }
    memcpy(&r, h + off, 4);
    return r;
}

}  // namespace avb

namespace avb {      // slots_hbd.cu: the 9 / 10-bit instances
static int slot_startcode(const uint8_t *buf, int size) { return startcode_find_candidate_cuda(buf, size); }
void h264dsp_init_hbd(H264DSPContext *c, int bits, int chroma_format_idc);
void h264qpel_init_hbd(H264QpelContext *c, int bits);
void h264chroma_init_hbd(H264ChromaContext *c, int bits);
}

using namespace avb;

// batched launchers reused as "batch of one"
extern "C" {
int ff_me_cmp_batch_cuda(int, int, int, const uint8_t *, const uint8_t *, ptrdiff_t, int, const FFMECmpRecord *, size_t, int32_t *, void *);
int ff_hpel_batch_cuda(const FFHpelRecord *, size_t, uint8_t *, const uint8_t *, ptrdiff_t, void *);
int ff_fdct_batch_cuda(int, int16_t *, size_t, void *);
int ff_mpeg4_qpel_batch_cuda(const FFQpelRecord *, size_t, uint8_t *, const uint8_t *, ptrdiff_t, void *);
int ff_pixblock_fdct_batch_cuda(int, const uint8_t *, const uint8_t *, const uint32_t *, const uint32_t *, ptrdiff_t, int16_t *, size_t, void *);
int ff_h264_weight_batch_cuda(const FFH264WeightRecord *, size_t, uint8_t *, const uint8_t *, int, void *);
}

namespace {

// ---- FDCT ----
template <int WHICH> void slot_fdct(int16_t *block)
{
    Stage S; if (!S.ok()) return;
    size_t o = S.take(128); memcpy(S.h + o, block, 128);
    if (S.up() || ff_fdct_batch_cuda(WHICH, (int16_t *)(S.d + o), 1, S.s) || S.down()) return;
    memcpy(block, S.h + o, 128);
}

// ---- Pixblock: get_pixels / diff_pixels as a batch of one (two staged 8x8 rectangles, pitch SP) ----
void slot_pixblock(int16_t *block, const uint8_t *s1, const uint8_t *s2, ptrdiff_t stride)
{
    Stage S; if (!S.ok()) return;
    const size_t o1 = S.rect_in(s1, stride, 8, 8), o2 = s2 ? S.rect_in(s2, stride, 8, 8) : 0, ob = S.take(128), oo = S.take(16);
    uint32_t *offs = (uint32_t *)(S.h + oo); offs[0] = (uint32_t)o1; offs[1] = (uint32_t)o2;
    if (S.up() || ff_pixblock_fdct_batch_cuda(-1, S.d, s2 ? S.d : nullptr, (const uint32_t *)(S.d + oo), (const uint32_t *)(S.d + oo) + 1, SP,
                                              (int16_t *)(S.d + ob), 1, S.s) || S.down()) return;
    memcpy(block, S.h + ob, 128);
}
void slot_get_pixels(int16_t *block, const uint8_t *pixels, ptrdiff_t stride) { slot_pixblock(block, pixels, nullptr, stride); }
void slot_diff_pixels(int16_t *block, const uint8_t *s1, const uint8_t *s2, ptrdiff_t stride) { slot_pixblock(block, s1, s2, stride); }

// ---- MECmp ----
template <int KIND, int SIDX, int DXY> int slot_mecmp(struct MpegEncContext *, uint8_t *a, uint8_t *b, ptrdiff_t stride, int h)
{
    Stage S; if (!S.ok()) return 0;
    const int w = SIDX == 0 ? 16 : SIDX == 1 ? 8 : 4;
    // exactly what the C function of this slot reads: one more column only for x2, one more row only for y2 (me_cmp.c:109-307) --
    // at the right / bottom edge of a frame without edge rows anything more lies outside the caller's buffer
    size_t oa = S.rect_in(a, stride, w, h), ob = S.rect_in(b, stride, w + (KIND == 0 ? DXY & 1 : 0), h + (KIND == 0 ? DXY >> 1 : 0)), orec = S.take(8), oout = S.take(16);
    memset(S.h + orec, 0, 8);
    if (S.up() || ff_me_cmp_batch_cuda(KIND, SIDX, DXY, S.d + oa, S.d + ob, SP, h, (const FFMECmpRecord *)(S.d + orec), 1, (int32_t *)(S.d + oout), S.s) || S.down()) return 0;
    int32_t r; memcpy(&r, S.h + oout, 4); return r;
}
int slot_sum_abs_dctelem(int16_t *block)
{
    Stage S; if (!S.ok()) return 0;
    size_t o = S.take(128), orec = S.take(8), oout = S.take(16);
    memcpy(S.h + o, block, 128); memset(S.h + orec, 0, 8);
    if (S.up() || ff_me_cmp_batch_cuda(10, 0, 0, S.d + o, S.d + o, 0, 0, (const FFMECmpRecord *)(S.d + orec), 1, (int32_t *)(S.d + oout), S.s) || S.down()) return 0;
    int32_t r; memcpy(&r, S.h + oout, 4); return r;
}

// ---- Hpel ----
template <int TAB, int SIDX, int DXY> void slot_hpel(uint8_t *block, const uint8_t *pixels, ptrdiff_t ls, int h)
{
    Stage S; if (!S.ok()) return;
    const int w = 16 >> SIDX;
    size_t od = S.rect_in(block, ls, w, h), os = S.rect_in(pixels, ls, w + (DXY & 1), h + (DXY >> 1)), orec = S.take(16);     // (hpeldsp.c:38-366 reads no more)
    FFHpelRecord r = { 0, 0, (uint8_t)TAB, (uint8_t)SIDX, (uint8_t)DXY, (uint8_t)h };
    memcpy(S.h + orec, &r, sizeof(r));
    if (S.up() || ff_hpel_batch_cuda((const FFHpelRecord *)(S.d + orec), 1, S.d + od, S.d + os, SP, S.s) || S.down()) return;
    S.rect_out(block, ls, w, h, od);
}

// ---- MPEG-4 qpel: stages exactly the rows / columns the C function of that phase reads ----
template <int KIND, int SIDX, int MC> void slot_mpeg4_qpel(uint8_t *dst, const uint8_t *src, ptrdiff_t stride)
{
    Stage S; if (!S.ok()) return;
    const int n = 16 >> SIDX, rows = (MC >> 2) ? n + 1 : n, cols = (MC & 3) ? n + 1 : n;
    size_t od = S.rect_in(dst, stride, n, n), os = S.rect_in(src, stride, cols, rows), orec = S.take(16);
    FFQpelRecord r = { 0, 0, (uint8_t)KIND, (uint8_t)SIDX, (uint8_t)MC, 0 };
    memcpy(S.h + orec, &r, sizeof(r));
    if (S.up() || ff_mpeg4_qpel_batch_cuda((const FFQpelRecord *)(S.d + orec), 1, S.d + od, S.d + os, SP, S.s) || S.down()) return;
    S.rect_out(dst, stride, n, n, od);
}
template <int KIND, int SIDX, int MC> struct FillMpeg4Qpel {
    static void go(qpel_mc_func *t) { t[MC] = slot_mpeg4_qpel<KIND, SIDX, MC>; FillMpeg4Qpel<KIND, SIDX, MC - 1>::go(t); }
};
template <int KIND, int SIDX> struct FillMpeg4Qpel<KIND, SIDX, -1> { static void go(qpel_mc_func *) {} };

// ---- H.264 qpel / chroma ----
template <int AVG, int SIDX, int MC> void slot_qpel(uint8_t *dst, const uint8_t *src, ptrdiff_t stride)
{
    Stage S; if (!S.ok()) return;
    const int n = 16 >> SIDX;
    size_t od = S.rect_in(dst, stride, n, n), os = S.rect_in(src - 2 * stride - 2, stride, n + 5, n + 5);
    SlotArgs a = {}; a.op = OP_H264_QPEL; a.a = AVG; a.b = n; a.c = MC; a.p0 = S.d + od; a.p1 = S.d + os + 2 * SP + 2;
    if (S.up() || S.run(a) || S.down()) return;
    S.rect_out(dst, stride, n, n, od);
}
template <int AVG, int WIDX> void slot_chroma(uint8_t *dst, uint8_t *src, ptrdiff_t stride, int h, int x, int y)
{
    Stage S; if (!S.ok()) return;
    const int w = 8 >> WIDX;
    // like the C code, the extra column / row is only read when its weight is non-zero
    size_t od = S.rect_in(dst, stride, w, h), os = S.rect_in(src, stride, w + (x != 0), h + (y != 0));
    SlotArgs a = {}; a.op = OP_H264_CHROMA_MC; a.a = AVG; a.b = w; a.c = h; a.d = x; a.e = y; a.p0 = S.d + od; a.p1 = S.d + os;
    if (S.up() || S.run(a) || S.down()) return;
    S.rect_out(dst, stride, w, h, od);
}

// ---- H264DSP ----
template <int WIDX> void slot_weight(uint8_t *block, int stride, int height, int log2_denom, int weight, int offset)
{
    Stage S; if (!S.ok()) return;
    const int w = 16 >> WIDX;
    size_t od = S.rect_in(block, stride, w, height), orec = S.take(16);
    FFH264WeightRecord r = { 0, (uint8_t)w, (uint8_t)height, (uint8_t)log2_denom, 0, (int16_t)weight, 0, (int16_t)offset, 0 };
    memcpy(S.h + orec, &r, sizeof(r));
    if (S.up() || ff_h264_weight_batch_cuda((const FFH264WeightRecord *)(S.d + orec), 1, S.d + od, nullptr, SP, S.s) || S.down()) return;
    S.rect_out(block, stride, w, height, od);
}
template <int WIDX> void slot_biweight(uint8_t *dst, uint8_t *src, int stride, int height, int log2_denom, int weightd, int weights, int offset)
{
    Stage S; if (!S.ok()) return;
    const int w = 16 >> WIDX;
    size_t od = S.rect_in(dst, stride, w, height), os = S.rect_in(src, stride, w, height), orec = S.take(16);
    FFH264WeightRecord r = { 0, (uint8_t)w, (uint8_t)height, (uint8_t)log2_denom, 0, (int16_t)weightd, (int16_t)weights, (int16_t)offset, 0 };
    memcpy(S.h + orec, &r, sizeof(r));
    if (S.up() || ff_h264_weight_batch_cuda((const FFH264WeightRecord *)(S.d + orec), 1, S.d + od, S.d + os, SP, S.s) || S.down()) return;
    S.rect_out(dst, stride, w, height, od);
}
// WHICH: 0 v_luma 1 h_luma 2 v_luma_intra 3 h_luma_intra 4 v_chroma 5 h_chroma 6 v_chroma_intra 7 h_chroma_intra, then the h_ variants
// that differ only in the lines per tc0 entry (h264dsp_template.c:158-163,222-229,272-283,314-328): 8 luma_mbaff 9 luma_mbaff_intra
// 10 chroma_mbaff 11 chroma_mbaff_intra 12 chroma422 13 chroma422_intra 14 chroma422_mbaff 15 chroma422_mbaff_intra
template <int WHICH> void loop_filter_impl(uint8_t *pix, int stride, int alpha, int beta, const int8_t *tc0)
{
    Stage S; if (!S.ok()) return;
    constexpr bool ext = WHICH >= 8;
    constexpr bool horiz_edge = !ext && !(WHICH & 1), chroma = ext ? WHICH >= 10 : WHICH >= 4, intra = ext ? (WHICH & 1) != 0 : (WHICH & 2) != 0;
    constexpr int ext_lines[8] = { 8, 8, 4, 4, 16, 16, 8, 8 };
    constexpr int lines = ext ? ext_lines[WHICH & 7] : chroma ? 8 : 16, reach = chroma ? 2 : 4;       // samples touched on each side of the edge
    const int w = horiz_edge ? lines : 2 * reach, h = horiz_edge ? 2 * reach : lines;
    uint8_t *org = horiz_edge ? pix - reach * stride : pix - reach;
    size_t o = S.rect_in(org, stride, w, h);
    SlotArgs a = {}; a.op = OP_H264_LOOP; a.a = (horiz_edge ? 1 : 0) | (chroma ? 2 : 0) | (intra ? 4 : 0); a.b = alpha; a.c = beta; a.d = lines;
    a.p0 = S.d + o + (horiz_edge ? reach * SP : reach);
    if (tc0) memcpy(a.tc0, tc0, 4);
    if (S.up() || S.run(a) || S.down()) return;
    S.rect_out(org, stride, w, h, o);
}
template <int WHICH> void slot_loop(uint8_t *pix, int stride, int alpha, int beta, int8_t *tc0) { loop_filter_impl<WHICH>(pix, stride, alpha, beta, tc0); }
template <int WHICH> void slot_loop_intra(uint8_t *pix, int stride, int alpha, int beta) { loop_filter_impl<WHICH>(pix, stride, alpha, beta, nullptr); }

template <int WHICH> void slot_h264_idct(uint8_t *dst, int16_t *block, int stride)
{
    Stage S; if (!S.ok()) return;
    const int n = (WHICH & 1) ? 8 : 4, coefs = (WHICH == 1) ? 64 : (WHICH == 0 ? 16 : 1);
    size_t od = S.rect_in(dst, stride, n, n), ob = S.take(128);
    memcpy(S.h + ob, block, (WHICH & 1) ? 128 : 32);
    SlotArgs a = {}; a.op = OP_H264_IDCT; a.a = WHICH; a.p0 = S.d + od; a.blk = (int16_t *)(S.d + ob);
    if (S.up() || S.run(a) || S.down()) return;
    S.rect_out(dst, stride, n, n, od);
    memcpy(block, S.h + ob, coefs * 2);                        // idct zeroes the block, dc_add only block[0]
}
// per-MB dispatchers: the caller's block_offset[] is honoured by staging the bounding rectangle of the blocks.
// WHICH: 0 add16, 1 add16intra, 2 idct8_add4, 3 add8 (4:2:0), 4 add8_422
template <int WHICH> void idct_mb_impl(uint8_t *dst, uint8_t **dst2, const int *bo, int16_t *block, int stride, const uint8_t *nnzc)
{
    Stage S; if (!S.ok()) return;
    if (stride <= 0) { set_error_msg("h264_idct_add16 slot", "non-positive stride is not taken over"); return; }
    constexpr int nb = WHICH == 2 ? 8 : 4, planes = WHICH >= 3 ? 2 : 1;
    constexpr int ncoef = (WHICH == 3 ? 36 : WHICH == 4 ? 40 : 16) * 16;       // coefficients up to the last block the C function may touch
    // the block_offset[] / scan8[] entries the C function reads
    int ent[16], n_ent = 0;
    if (WHICH <= 1) for (int i = 0; i < 16; i++) ent[n_ent++] = i;
    else if (WHICH == 2) for (int i = 0; i < 16; i += 4) ent[n_ent++] = i;
    else for (int p = 0; p < 2; p++) for (int k = 0; k < (WHICH == 4 ? 8 : 4); k++) ent[n_ent++] = 16 + 16 * p + (k >= 4 ? k + 4 : k);
    int W = 0, H = 0;
    for (int n = 0; n < n_ent; n++) {
        const int i = ent[n];
        if (bo[i] < 0) { set_error_msg("h264_idct_add16 slot", "negative block offsets are not taken over"); return; }
        int x = bo[i] % stride + nb, y = bo[i] / stride + nb;
        if (x > W) W = x;
        if (y > H) H = y;
    }
    const int pitch = (W + 15) & ~15;
    if ((size_t)pitch * H * planes + 2048 > Stage::CAP) { set_error_msg("h264_idct_add16 slot", "block offsets span too large a rectangle"); return; }
    size_t od[2];
    for (int p = 0; p < planes; p++) {
        od[p] = S.take((size_t)pitch * H);
        const uint8_t *src = WHICH >= 3 ? dst2[p] : dst;
        for (int y = 0; y < H; y++) memcpy(S.h + od[p] + (size_t)y * pitch, src + (size_t)y * stride, W);
    }
    size_t ob = S.take(48 * 16 * 2);
    memcpy(S.h + ob, block, ncoef * 2);
    SlotArgs a = {}; a.op = OP_H264_IDCT_MB; a.a = WHICH; a.b = pitch; a.p0 = S.d + od[0]; a.p1 = planes == 2 ? S.d + od[1] : nullptr;
    a.blk = (int16_t *)(S.d + ob);
    for (int i = 0; i < 48; i++) a.off[i] = 0;
    for (int n = 0; n < n_ent; n++) { const int i = ent[n]; a.off[i] = (bo[i] / stride) * pitch + bo[i] % stride; }
    memcpy(a.nnzc, nnzc, 120);
    if (S.up() || S.run(a) || S.down()) return;
    for (int p = 0; p < planes; p++) {
        uint8_t *d = WHICH >= 3 ? dst2[p] : dst;
        for (int y = 0; y < H; y++) memcpy(d + (size_t)y * stride, S.h + od[p] + (size_t)y * pitch, W);
    }
    memcpy(block, S.h + ob, ncoef * 2);
}
template <int WHICH> void slot_idct_mb(uint8_t *dst, const int *bo, int16_t *block, int stride, const uint8_t nnzc[15 * 8]) { idct_mb_impl<WHICH>(dst, nullptr, bo, block, stride, nnzc); }
template <int WHICH> void slot_idct_add8(uint8_t **dst, const int *bo, int16_t *block, int stride, const uint8_t nnzc[15 * 8]) { idct_mb_impl<WHICH>(nullptr, dst, bo, block, stride, nnzc); }

void slot_luma_dc(int16_t *output, int16_t *input, int qmul)
{
    Stage S; if (!S.ok()) return;
    size_t o = S.take(512 + 32);
    memcpy(S.h + o, output, 512); memcpy(S.h + o + 512, input, 32);        // output holds the MB's 16 blocks of 16
    SlotArgs a = {}; a.op = OP_H264_LUMA_DC; a.a = qmul; a.blk = (int16_t *)(S.d + o);
    if (S.up() || S.run(a) || S.down()) return;
    memcpy(output, S.h + o, 512);
}
// C422 = 0: the 2x2 transform touches block[0 / 16 / 32 / 48]; C422 = 1: the 2x4 transform touches block[16 k], k < 8
template <int C422> void slot_chroma_dc(int16_t *block, int qmul)
{
    Stage S; if (!S.ok()) return;
    constexpr size_t bytes = C422 ? 113 * 2 : 128;
    size_t o = S.take(256);
    memcpy(S.h + o, block, bytes);
    SlotArgs a = {}; a.op = OP_H264_CHROMA_DC; a.a = qmul; a.b = C422; a.blk = (int16_t *)(S.d + o);
    if (S.up() || S.run(a) || S.down()) return;
    memcpy(block, S.h + o, bytes);
}
template <int N> void slot_add_pixels_clear(uint8_t *dst, int16_t *block, int stride)
{
    Stage S; if (!S.ok()) return;
    size_t od = S.rect_in(dst, stride, N, N), ob = S.take(128);
    memcpy(S.h + ob, block, N * N * 2);
    SlotArgs a = {}; a.op = OP_H264_ADD_PIXELS; a.a = N; a.p0 = S.d + od; a.blk = (int16_t *)(S.d + ob);
    if (S.up() || S.run(a) || S.down()) return;
    S.rect_out(dst, stride, N, N, od);
    memcpy(block, S.h + ob, N * N * 2);
}

template <int AVG, int SIDX> void fill_qpel(qpel_mc_func *t)
{
#define Q(mc) t[mc] = slot_qpel<AVG, SIDX, mc>;
    Q(0) Q(1) Q(2) Q(3) Q(4) Q(5) Q(6) Q(7) Q(8) Q(9) Q(10) Q(11) Q(12) Q(13) Q(14) Q(15)
#undef Q
}
template <int TAB, int SIDX> void fill_hpel(op_pixels_func *t)
{
    t[0] = slot_hpel<TAB, SIDX, 0>; t[1] = slot_hpel<TAB, SIDX, 1>; t[2] = slot_hpel<TAB, SIDX, 2>; t[3] = slot_hpel<TAB, SIDX, 3>;
}

}  // namespace

extern "C" {

void ff_qpeldsp_init_cuda(QpelDSPContext *c)
{
    avb::enter();
    if (!c) return;
    FillMpeg4Qpel<0, 0, 15>::go(c->put_qpel_pixels_tab[0]);        FillMpeg4Qpel<0, 1, 15>::go(c->put_qpel_pixels_tab[1]);
    FillMpeg4Qpel<1, 0, 15>::go(c->put_no_rnd_qpel_pixels_tab[0]); FillMpeg4Qpel<1, 1, 15>::go(c->put_no_rnd_qpel_pixels_tab[1]);
    FillMpeg4Qpel<2, 0, 15>::go(c->avg_qpel_pixels_tab[0]);        FillMpeg4Qpel<2, 1, 15>::go(c->avg_qpel_pixels_tab[1]);
}

void ff_pixblockdsp_init_cuda(PixblockDSPContext *c, unsigned high_bit_depth)
{
    avb::enter();
    if (!c || high_bit_depth) return;
    c->get_pixels = slot_get_pixels; c->diff_pixels = slot_diff_pixels;
}

void ff_fdctdsp_init_cuda(FDCTDSPContext *c, int dct_algo, int bits_per_raw_sample, unsigned high_bit_depth)
{
    avb::enter();
    if (bits_per_raw_sample == 10) { c->fdct = slot_fdct<4>; c->fdct248 = slot_fdct<5>; return; }      // fdctdsp.c:31-33: the 10-bit islow pair whatever dct_algo says
    if (high_bit_depth || bits_per_raw_sample > 8) return;               // other depths: the reference falls through to its 8-bit functions; not taken over
    if (dct_algo == AVB_FF_DCT_FASTINT) { c->fdct = slot_fdct<2>; c->fdct248 = slot_fdct<3>; }
    else if (dct_algo == AVB_FF_DCT_AUTO || dct_algo == AVB_FF_DCT_INT) { c->fdct = slot_fdct<0>; c->fdct248 = slot_fdct<1>; }
    else if (dct_algo == AVB_FF_DCT_FAAN) { c->fdct = slot_fdct<6>; c->fdct248 = slot_fdct<7>; }
}

void ff_me_cmp_init_cuda(MECmpContext *c)
{
    avb::enter();
    // mirrors the assignments of ff_me_cmp_init (libavcodec/me_cmp.c:895-944); slots that need encoder state
    // (dct_sad, dct_max, dct264_sad, quant_psnr, rd, bit) keep whatever the caller installed
    c->sum_abs_dctelem = slot_sum_abs_dctelem;
    c->pix_abs[0][0] = slot_mecmp<0, 0, 0>; c->pix_abs[0][1] = slot_mecmp<0, 0, 1>; c->pix_abs[0][2] = slot_mecmp<0, 0, 2>; c->pix_abs[0][3] = slot_mecmp<0, 0, 3>;
    c->pix_abs[1][0] = slot_mecmp<0, 1, 0>; c->pix_abs[1][1] = slot_mecmp<0, 1, 1>; c->pix_abs[1][2] = slot_mecmp<0, 1, 2>; c->pix_abs[1][3] = slot_mecmp<0, 1, 3>;
    c->sad[0] = slot_mecmp<1, 0, 0>; c->sad[1] = slot_mecmp<1, 1, 0>;
    c->sse[0] = slot_mecmp<2, 0, 0>; c->sse[1] = slot_mecmp<2, 1, 0>; c->sse[2] = slot_mecmp<2, 2, 0>;
    c->hadamard8_diff[0] = slot_mecmp<3, 0, 0>; c->hadamard8_diff[1] = slot_mecmp<3, 1, 0>;
    c->hadamard8_diff[4] = slot_mecmp<7, 0, 0>; c->hadamard8_diff[5] = slot_mecmp<7, 1, 0>;
    c->vsad[0] = slot_mecmp<4, 0, 0>; c->vsad[4] = slot_mecmp<8, 0, 0>; c->vsad[5] = slot_mecmp<8, 1, 0>;
    c->vsse[0] = slot_mecmp<5, 0, 0>; c->vsse[4] = slot_mecmp<9, 0, 0>; c->vsse[5] = slot_mecmp<9, 1, 0>;
    c->nsse[0] = slot_mecmp<6, 0, 0>; c->nsse[1] = slot_mecmp<6, 1, 0>;
}

void ff_h264dsp_init_cuda(H264DSPContext *c, const int bit_depth, const int chroma_format_idc)
{
    avb::enter();
    if (bit_depth == 9 || bit_depth == 10) { h264dsp_init_hbd(c, bit_depth, chroma_format_idc); c->startcode_find_candidate = slot_startcode; return; }
    if (bit_depth != 8) return;                                           // other depths do not exist for H.264 here (h264dsp.c:126-136 maps them to 8)
    const bool c420 = chroma_format_idc <= 1;                             // the reference's own test, h264dsp.c:81-122
    c->weight_h264_pixels_tab[0] = slot_weight<0>; c->weight_h264_pixels_tab[1] = slot_weight<1>;
    c->weight_h264_pixels_tab[2] = slot_weight<2>; c->weight_h264_pixels_tab[3] = slot_weight<3>;
    c->biweight_h264_pixels_tab[0] = slot_biweight<0>; c->biweight_h264_pixels_tab[1] = slot_biweight<1>;
    c->biweight_h264_pixels_tab[2] = slot_biweight<2>; c->biweight_h264_pixels_tab[3] = slot_biweight<3>;
    c->h264_v_loop_filter_luma = slot_loop<0>; c->h264_h_loop_filter_luma = slot_loop<1>;
    c->h264_h_loop_filter_luma_mbaff = slot_loop<8>;
    c->h264_v_loop_filter_luma_intra = slot_loop_intra<2>; c->h264_h_loop_filter_luma_intra = slot_loop_intra<3>;
    c->h264_h_loop_filter_luma_mbaff_intra = slot_loop_intra<9>;
    c->h264_v_loop_filter_chroma = slot_loop<4>;
    c->h264_h_loop_filter_chroma = c420 ? slot_loop<5> : slot_loop<12>;
    c->h264_h_loop_filter_chroma_mbaff = c420 ? slot_loop<10> : slot_loop<14>;
    c->h264_v_loop_filter_chroma_intra = slot_loop_intra<6>;
    c->h264_h_loop_filter_chroma_intra = c420 ? slot_loop_intra<7> : slot_loop_intra<13>;
    c->h264_h_loop_filter_chroma_mbaff_intra = c420 ? slot_loop_intra<11> : slot_loop_intra<15>;
    // h264_loop_filter_strength stays NULL like in C (h264dsp.c:124)
    c->startcode_find_candidate = slot_startcode;                         // h264dsp.c:137, every bit depth
    c->h264_idct_add = slot_h264_idct<0>; c->h264_idct8_add = slot_h264_idct<1>;
    c->h264_idct_dc_add = slot_h264_idct<2>; c->h264_idct8_dc_add = slot_h264_idct<3>;
    c->h264_idct_add16 = slot_idct_mb<0>; c->h264_idct_add16intra = slot_idct_mb<1>; c->h264_idct8_add4 = slot_idct_mb<2>;
    c->h264_idct_add8 = c420 ? slot_idct_add8<3> : slot_idct_add8<4>;
    c->h264_luma_dc_dequant_idct = slot_luma_dc;
    c->h264_chroma_dc_dequant_idct = c420 ? slot_chroma_dc<0> : slot_chroma_dc<1>;
    c->h264_add_pixels8_clear = slot_add_pixels_clear<8>; c->h264_add_pixels4_clear = slot_add_pixels_clear<4>;
}

void ff_h264qpel_init_cuda(H264QpelContext *c, int bit_depth)
{
    avb::enter();
    if (bit_depth == 9 || bit_depth == 10) { h264qpel_init_hbd(c, bit_depth); return; }
    if (bit_depth != 8) return;
    fill_qpel<0, 0>(c->put_h264_qpel_pixels_tab[0]); fill_qpel<0, 1>(c->put_h264_qpel_pixels_tab[1]);
    fill_qpel<0, 2>(c->put_h264_qpel_pixels_tab[2]); fill_qpel<0, 3>(c->put_h264_qpel_pixels_tab[3]);
    fill_qpel<1, 0>(c->avg_h264_qpel_pixels_tab[0]); fill_qpel<1, 1>(c->avg_h264_qpel_pixels_tab[1]);
    fill_qpel<1, 2>(c->avg_h264_qpel_pixels_tab[2]);             // the reference has no avg 2x2 row (h264qpel.c:60-67)
}

void ff_h264chroma_init_cuda(H264ChromaContext *c, int bit_depth)
{
    avb::enter();
    if (bit_depth == 9 || bit_depth == 10) { h264chroma_init_hbd(c, bit_depth); return; }
    if (bit_depth != 8) return;
    c->put_h264_chroma_pixels_tab[0] = slot_chroma<0, 0>; c->put_h264_chroma_pixels_tab[1] = slot_chroma<0, 1>; c->put_h264_chroma_pixels_tab[2] = slot_chroma<0, 2>;
    c->avg_h264_chroma_pixels_tab[0] = slot_chroma<1, 0>; c->avg_h264_chroma_pixels_tab[1] = slot_chroma<1, 1>; c->avg_h264_chroma_pixels_tab[2] = slot_chroma<1, 2>;
}

void ff_hpeldsp_init_cuda(HpelDSPContext *c, int flags)
{
    avb::enter();
    (void)flags;
    fill_hpel<0, 0>(c->put_pixels_tab[0]); fill_hpel<0, 1>(c->put_pixels_tab[1]); fill_hpel<0, 2>(c->put_pixels_tab[2]); fill_hpel<0, 3>(c->put_pixels_tab[3]);
    fill_hpel<1, 0>(c->avg_pixels_tab[0]); fill_hpel<1, 1>(c->avg_pixels_tab[1]); fill_hpel<1, 2>(c->avg_pixels_tab[2]); fill_hpel<1, 3>(c->avg_pixels_tab[3]);
    fill_hpel<2, 0>(c->put_no_rnd_pixels_tab[0]); fill_hpel<2, 1>(c->put_no_rnd_pixels_tab[1]);      // [2], [3] are NULL in C too (hpeldsp.c:352-353)
    fill_hpel<3, 0>(c->avg_no_rnd_pixels_tab);
}

}  // extern "C"
