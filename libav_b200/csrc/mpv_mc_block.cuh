// libav_b200/csrc/mpv_mc_block.cuh -- ff_mpv_motion() (libavcodec/mpegvideo_motion.c:814-968) for one macroblock, one lane per
// destination column: lanes 0-15 own the 16 luma columns, 16-23 the cb columns, 24-31 the cr columns (4:4:4: a 48-column map, lane l
// owning columns l and l + 32).  Each lane walks the record exactly as the C code does (same vector derivations, clips, edge tests and
// call order) and runs every pixel operation only on its own column, reading the destination back where the operation is an avg.  Lanes
// never communicate, so tests/hostsim/ compiles this file as host C++ and the CPU suite checks it against the reference.
//
// The body is a template over the picture kind: CF, the chroma format (1 4:2:0, 2 4:2:2, 3 4:4:4; MPEG-1 / MPEG-2 only beyond 1), and IL,
// an interlaced H.263-family picture (FIELD records taken, edge emulation in frame rows).  CF 1, IL 0 is the progressive 4:2:0 body every
// other picture runs; each other kind runs in launches of its own (mpv_mc.cu).
#pragma once
#include "common.cuh"
#include "../../include/avdsp_b200.h"

namespace avb {

enum { MPV_MC_16X16 = 0, MPV_MC_8X8 = 1, MPV_MC_16X8 = 2, MPV_MC_FIELD = 3, MPV_MC_DMV = 4 };
enum { MPV_PICT_TOP = 1, MPV_PICT_BOTTOM = 2, MPV_PICT_FRAME = 3 };
enum { MPV_BUG_QPEL_CHROMA = 64, MPV_BUG_QPEL_CHROMA2 = 256, MPV_BUG_HPEL_CHROMA = 2048 };

// what the kernel reads of one picture (filled and checked by ff_mpv_motion_batch_cuda)
struct MpvMcPic {
    uint8_t *dest[3];
    const uint8_t *cur[3], *ref[2][3];
    int ls[2];             // s->linesize, s->uvlinesize
    int pic_k;             // current_picture.f->linesize / s->linesize: 1 frame picture, 2 field picture
    int mb_w, mb_rows;     // macroblocks per row, macroblock rows of the picture (a field has mb_height / 2)
    int width, height, h_edge, v_edge;
    int h263, structure, first_field, b_pic, no_rnd, bugs, qpel;
    int rw[2], rh[2];      // readable region of a reference plane: columns [0, rw), frame rows [0, rh) (luma, chroma)
};

// the source of one pixel operation: sample (x, y) of the operation is read at picture position (x0 + x, y0 + y), clamped to
// [0, ew) x [0, eh) when the reference emulates the edge, then at frame row y * k + f (k: row step, f: field_select).  In an interlaced
// picture (IL) the row is clamped after that step, to frame rows [0, eh): emulated_edge_mc copies a frame window from row 2 * src_y
// and field_select then picks every other line of it (mpegvideo_motion.c:226-256, :355-359)
struct MpvSrc {
    const uint8_t *base;
    int x0, y0, k, f, emu, ew, eh;
};

struct MpvLane {
    int pl, c;             // plane 0 / 1 / 2, column inside the macroblock
    uint8_t *dcol;         // destination sample of row 0 of the macroblock in this column
    ptrdiff_t dls;         // destination row pitch: the picture's linesize
};

__device__ __forceinline__ int mpv_fetch_frame_rows(const MpvMcPic &P, int pl, const MpvSrc &s, int x, int y)
{
    x += s.x0;
    y = (y + s.y0) * s.k + s.f;
    if (s.emu) { x = min(max(x, 0), s.ew - 1); y = min(max(y, 0), s.eh - 1); }
    const int c = pl != 0;
    const int r = min(max(y, 0), P.rh[c] - 1);
    x = min(max(x, 0), P.rw[c] - 1);
    return s.base[(ptrdiff_t)r * P.ls[c] + x];
}

template <int IL = 0>
__device__ __forceinline__ int mpv_fetch(const MpvMcPic &P, int pl, const MpvSrc &s, int x, int y)
{
    if (IL) return mpv_fetch_frame_rows(P, pl, s, x, y);
    x += s.x0; y += s.y0;
    if (s.emu) { x = min(max(x, 0), s.ew - 1); y = min(max(y, 0), s.eh - 1); }
    const int c = pl != 0;
    // the readable region: the C code never reads outside it, so this clamp only ever acts on records it would misread
    const int r = min(max(y * s.k + s.f, 0), P.rh[c] - 1);
    x = min(max(x, 0), P.rw[c] - 1);
    return s.base[(ptrdiff_t)r * P.ls[c] + x];
}

__device__ __forceinline__ void mpv_store(const MpvLane &L, int row, int v, int avg)
{
    uint8_t *o = L.dcol + row * L.dls;
    *o = (uint8_t)(avg ? (*o + v + 1) >> 1 : v);      // op_avg = rnd_avg32 (hpeldsp_template.c, qpeldsp.c)
}

// HpelDSPContext put / put_no_rnd / avg pixels (hpeldsp_template.c): w x h block whose destination rows are r0 + i * rstep
template <int IL = 0>
__device__ __forceinline__ void mpv_hpel(const MpvMcPic &P, const MpvLane &L, int pl, int c0, int w, int r0, int rstep, int h,
                                         const MpvSrc &s, int dxy, int no_rnd, int avg)
{
    if (L.pl != pl || L.c < c0 || L.c >= c0 + w) return;
    const int j = L.c - c0;
    for (int i = 0; i < h; i++) {
        const int a = mpv_fetch<IL>(P, pl, s, j, i);
        int v;
        if (dxy == 0)      v = a;
        else if (dxy == 1) v = (a + mpv_fetch<IL>(P, pl, s, j + 1, i) + 1 - no_rnd) >> 1;
        else if (dxy == 2) v = (a + mpv_fetch<IL>(P, pl, s, j, i + 1) + 1 - no_rnd) >> 1;
        else v = (a + mpv_fetch<IL>(P, pl, s, j + 1, i) + mpv_fetch<IL>(P, pl, s, j, i + 1) + mpv_fetch<IL>(P, pl, s, j + 1, i + 1) + 2 - no_rnd) >> 2;
        mpv_store(L, r0 + i * rstep, v, avg);
    }
}

// the MPEG-4 8-tap half-sample filter (qpeldsp.c mpeg4_qpel*_h/v_lowpass) at position i of an N-sample line, indices mirrored at both
// ends of the block; t(j) reads sample j
template <int N, class T>
__device__ __forceinline__ int mpv_qpel_tap(T t, int i, int rnd)
{
    auto m = [](int j) { return j < 0 ? -1 - j : j > N ? 2 * N + 1 - j : j; };
    const int v = (t(m(i)) + t(m(i + 1))) * 20 - (t(m(i - 1)) + t(m(i + 2))) * 6 + (t(m(i - 2)) + t(m(i + 3))) * 3 - (t(m(i - 3)) + t(m(i + 4)));
    return clip_u8((v + rnd) >> 5);
}

// QpelDSPContext put / put_no_rnd / avg qpel pixels (qpeldsp.c:39-700) for one N x N block at (c0, r0) of the luma macroblock: every
// quarter-sample position as the C code composes it -- the horizontal phase plane (full-sample, half-sample, or their rounded mean),
// then the same along the columns of that plane.  The lane computes its column of the plane only.
template <int N, int IL = 0>
__device__ __forceinline__ void mpv_qpel(const MpvMcPic &P, const MpvLane &L, int c0, int r0, const MpvSrc &s, int mc, int no_rnd, int avg)
{
    if (L.pl != 0 || L.c < c0 || L.c >= c0 + N) return;
    const int j = L.c - c0, x = mc & 3, y = mc >> 2, rnd = no_rnd ? 15 : 16, up = no_rnd ? 0 : 1;
    int hx[N + 1];
#pragma unroll
    for (int rr = 0; rr <= N; rr++) {
        if (rr == N && !y) break;
        int v = mpv_fetch<IL>(P, 0, s, j + (x == 3), rr);
        if (x) {
            const int h = mpv_qpel_tap<N>([&](int cc) { return mpv_fetch<IL>(P, 0, s, cc, rr); }, j, rnd);
            v = x == 2 ? h : (v + h + up) >> 1;
        }
        hx[rr] = v;
    }
#pragma unroll
    for (int i = 0; i < N; i++) {
        int v = hx[i];
        if (y) {
            const int vv = mpv_qpel_tap<N>([&](int rr) { return hx[rr]; }, i, rnd);
            v = y == 2 ? vv : ((y == 3 ? hx[i + 1] : hx[i]) + vv + up) >> 1;
        }
        mpv_store(L, r0 + i, v, avg);
    }
}

// mpeg_motion_internal (mpegvideo_motion.c:258-373): one vector onto the three planes.  r0: first destination row of the luma part
// inside the macroblock, before the bottom_field step.  Returns without touching anything where the C code does.
template <int CF = 1, int IL = 0>
__device__ __forceinline__ void mpv_mpeg_motion(const MpvMcPic &P, const MpvLane &L, const FFMpvMCRecord &r, int field_based, int bottom,
                                                int field_select, const uint8_t *const *ref, int no_rnd, int avg, int mx, int my, int h,
                                                int mb_y, int r0)
{
    const int v_edge = P.v_edge >> field_based;
    const int dxy = ((my & 1) << 1) | (mx & 1);
    const int src_x = r.mb_x * 16 + (mx >> 1), src_y = (mb_y << (4 - field_based)) + (my >> 1);
    int uvdxy, uvsrc_x, uvsrc_y;
    if (P.h263) {
        if (IL && field_based && (P.bugs & MPV_BUG_HPEL_CHROMA)) {   // field_based only in interlaced pictures
            const int cmx = (mx >> 1) | (mx & 1), cmy = my >> 1;
            uvdxy = ((cmy & 1) << 1) | (cmx & 1);
            uvsrc_x = r.mb_x * 8 + (cmx >> 1);
            uvsrc_y = (mb_y << (3 - field_based)) + (cmy >> 1);
        } else {
            uvdxy = dxy | (my & 2) | ((mx & 2) >> 1);
            uvsrc_x = src_x >> 1;
            uvsrc_y = src_y >> 1;
        }
    } else if (CF == 1) {
        const int cmx = mx / 2, cmy = my / 2;              // C truncation
        uvdxy = ((cmy & 1) << 1) | (cmx & 1);
        uvsrc_x = r.mb_x * 8 + (cmx >> 1);
        uvsrc_y = (mb_y << (3 - field_based)) + (cmy >> 1);
    } else if (CF == 2) {
        const int cmx = mx / 2;
        uvdxy = ((my & 1) << 1) | (cmx & 1);
        uvsrc_x = r.mb_x * 8 + (cmx >> 1);
        uvsrc_y = src_y;
    } else {
        uvdxy = dxy;
        uvsrc_x = src_x;
        uvsrc_y = src_y;
    }
    int emu = 0;
    if ((unsigned)src_x > (unsigned)max(P.h_edge - (mx & 1) - 16, 0) || (unsigned)src_y > (unsigned)max(v_edge - (my & 1) - h, 0)) {
        if (!P.h263) return;                               // "MPEG motion vector out of boundary": the call is skipped
        emu = 1;
    }
    const int k = P.pic_k << field_based, rstep = 1 << field_based;
    const int cx = CF != 3, cy = CF == 1;                  // chroma_x_shift, chroma_y_shift
    const MpvSrc sy = { ref[0], src_x, src_y, k, field_select, emu, P.h_edge, P.v_edge };
    mpv_hpel<IL>(P, L, 0, 0, 16, r0 + bottom, rstep, h, sy, dxy, no_rnd, avg);
    for (int p = 1; p < 3; p++) {
        const MpvSrc sc = { ref[p], uvsrc_x, uvsrc_y, k, field_select, emu, P.h_edge >> 1, P.v_edge >> 1 };
        mpv_hpel<IL>(P, L, p, 0, 16 >> cx, (r0 >> cy) + bottom, rstep, h >> cy, sc, uvdxy, no_rnd, avg);
    }
}

// qpel_motion (mpegvideo_motion.c:492-572), frame-based
__device__ __forceinline__ void mpv_qpel_motion(const MpvMcPic &P, const MpvLane &L, const FFMpvMCRecord &r, const uint8_t *const *ref,
                                                int no_rnd, int avg, int mx, int my)
{
    const int dxy = ((my & 3) << 2) | (mx & 3);
    const int src_x = r.mb_x * 16 + (mx >> 2), src_y = r.mb_y * 16 + (my >> 2);
    int cmx, cmy;
    if (P.bugs & MPV_BUG_QPEL_CHROMA2) {
        // rtab[8] = { 0, 0, 1, 1, 0, 0, 0, 1 } as a bit mask
        cmx = (mx >> 1) + ((0x8C >> (mx & 7)) & 1);
        cmy = (my >> 1) + ((0x8C >> (my & 7)) & 1);
    } else if (P.bugs & MPV_BUG_QPEL_CHROMA) {
        cmx = (mx >> 1) | (mx & 1);
        cmy = (my >> 1) | (my & 1);
    } else {
        cmx = mx / 2;
        cmy = my / 2;
    }
    cmx = (cmx >> 1) | (cmx & 1);
    cmy = (cmy >> 1) | (cmy & 1);
    const int uvdxy = (cmx & 1) | ((cmy & 1) << 1);
    cmx >>= 1;
    cmy >>= 1;
    const int emu = (unsigned)src_x > (unsigned)max(P.h_edge - (mx & 3) - 16, 0) || (unsigned)src_y > (unsigned)max(P.v_edge - (my & 3) - 16, 0);
    const MpvSrc sy = { ref[0], src_x, src_y, 1, 0, emu, P.h_edge, P.v_edge };
    mpv_qpel<16>(P, L, 0, 0, sy, dxy, no_rnd, avg);
    for (int p = 1; p < 3; p++) {
        const MpvSrc sc = { ref[p], r.mb_x * 8 + cmx, r.mb_y * 8 + cmy, 1, 0, emu, P.h_edge >> 1, P.v_edge >> 1 };
        mpv_hpel(P, L, p, 0, 8, 0, 1, 8, sc, uvdxy, no_rnd, avg);
    }
}

// qpel_motion with field_based (mpegvideo_motion.c:492-572), interlaced MPEG-4 only: one field of the macroblock, its luma as two 8x8 qpel
// ops (mirrored at the 8-sample block edges) on field lines, chroma from mx / 2, my >> 1 (no QPEL_CHROMA workaround) over 4 field lines
__device__ __forceinline__ void mpv_qpel_field(const MpvMcPic &P, const MpvLane &L, const FFMpvMCRecord &r, int bottom, int field_select,
                                               const uint8_t *const *ref, int no_rnd, int avg, int mx, int my)
{
    const int dxy = ((my & 3) << 2) | (mx & 3);
    const int src_x = r.mb_x * 16 + (mx >> 2), src_y = r.mb_y * 8 + (my >> 2);
    int cmx = mx / 2, cmy = my >> 1;
    cmx = (cmx >> 1) | (cmx & 1);
    cmy = (cmy >> 1) | (cmy & 1);
    const int uvdxy = (cmx & 1) | ((cmy & 1) << 1);
    cmx >>= 1;
    cmy >>= 1;
    const int emu = (unsigned)src_x > (unsigned)max(P.h_edge - (mx & 3) - 16, 0) ||
                    (unsigned)src_y > (unsigned)max((P.v_edge >> 1) - (my & 3) - 8, 0);
    MpvLane F = L;                                         // the field's lines: one line down for the bottom field, every other line
    F.dcol += bottom * L.dls;
    F.dls = 2 * L.dls;
    for (int b = 0; b < 2; b++) {
        const MpvSrc sy = { ref[0], src_x + 8 * b, src_y, 2, field_select, emu, P.h_edge, P.v_edge };
        mpv_qpel<8, 1>(P, F, 8 * b, 0, sy, dxy, no_rnd, avg);
    }
    for (int p = 1; p < 3; p++) {
        const MpvSrc sc = { ref[p], r.mb_x * 8 + cmx, r.mb_y * 4 + cmy, 2, field_select, emu, P.h_edge >> 1, P.v_edge >> 1 };
        mpv_hpel<1>(P, F, p, 0, 8, 0, 1, 4, sc, uvdxy, no_rnd, avg);
    }
}

// chroma_4mv_motion (mpegvideo_motion.c:577-627): the one chroma vector of a 4MV macroblock, from the sum of its four luma vectors
__device__ __forceinline__ void mpv_chroma_4mv(const MpvMcPic &P, const MpvLane &L, const FFMpvMCRecord &r, const uint8_t *const *ref,
                                               int no_rnd, int avg, int mx, int my)
{
    // ff_h263_round_chroma (motion_est.h:96-104); its table { 0, 0, 0, 1, 1, 1, 1, 1, 0, 0, 0, 0, 0, 0, 1, 1 } as a bit mask
    mx = ((0xC0F8 >> (mx & 0xf)) & 1) + (mx >> 3);
    my = ((0xC0F8 >> (my & 0xf)) & 1) + (my >> 3);
    int dxy = ((my & 1) << 1) | (mx & 1);
    mx >>= 1;
    my >>= 1;
    int src_x = r.mb_x * 8 + mx, src_y = r.mb_y * 8 + my;
    src_x = min(max(src_x, -8), P.width >> 1);
    if (src_x == (P.width >> 1)) dxy &= ~1;
    src_y = min(max(src_y, -8), P.height >> 1);
    if (src_y == (P.height >> 1)) dxy &= ~2;
    const int emu = (unsigned)src_x > (unsigned)max((P.h_edge >> 1) - (dxy & 1) - 8, 0) ||
                    (unsigned)src_y > (unsigned)max((P.v_edge >> 1) - (dxy >> 1) - 8, 0);
    for (int p = 1; p < 3; p++) {
        const MpvSrc sc = { ref[p], src_x, src_y, 1, 0, emu, P.h_edge >> 1, P.v_edge >> 1 };
        mpv_hpel(P, L, p, 0, 8, 0, 1, 8, sc, dxy, no_rnd, avg);
    }
}

// apply_8x8 (mpegvideo_motion.c:730-800): four 8x8 luma vectors (hpel_motion, :192-224, or the quarter-sample loop) and chroma_4mv_motion
__device__ __forceinline__ void mpv_apply_8x8(const MpvMcPic &P, const MpvLane &L, const FFMpvMCRecord &r, int dir, const uint8_t *const *ref,
                                              int no_rnd, int avg)
{
    int cmx = 0, cmy = 0;
    for (int i = 0; i < 4; i++) {
        const int mx = r.mv[dir][i][0], my = r.mv[dir][i][1];
        int dxy, src_x, src_y, emu;
        if (P.qpel) {
            dxy = ((my & 3) << 2) | (mx & 3);
            src_x = r.mb_x * 16 + (mx >> 2) + (i & 1) * 8;
            src_y = r.mb_y * 16 + (my >> 2) + (i >> 1) * 8;
            src_x = min(max(src_x, -16), P.width);
            if (src_x == P.width) dxy &= ~3;
            src_y = min(max(src_y, -16), P.height);
            if (src_y == P.height) dxy &= ~12;
            emu = (unsigned)src_x > (unsigned)max(P.h_edge - (mx & 3) - 8, 0) || (unsigned)src_y > (unsigned)max(P.v_edge - (my & 3) - 8, 0);
            cmx += mx / 2;
            cmy += my / 2;
        } else {
            dxy = 0;
            src_x = r.mb_x * 16 + (i & 1) * 8 + (mx >> 1);
            src_y = r.mb_y * 16 + (i >> 1) * 8 + (my >> 1);
            src_x = min(max(src_x, -16), P.width);
            if (src_x != P.width) dxy |= mx & 1;
            src_y = min(max(src_y, -16), P.height);
            if (src_y != P.height) dxy |= (my & 1) << 1;
            emu = (unsigned)src_x > (unsigned)max(P.h_edge - (mx & 1) - 8, 0) || (unsigned)src_y > (unsigned)max(P.v_edge - (my & 1) - 8, 0);
            cmx += mx;
            cmy += my;
        }
        const MpvSrc s = { ref[0], src_x, src_y, 1, 0, emu, P.h_edge, P.v_edge };
        if (P.qpel) mpv_qpel<8>(P, L, (i & 1) * 8, (i >> 1) * 8, s, dxy, no_rnd, avg);
        else        mpv_hpel(P, L, 0, (i & 1) * 8, 8, (i >> 1) * 8, 1, 8, s, dxy, no_rnd, avg);
    }
    mpv_chroma_4mv(P, L, r, ref, no_rnd, avg, cmx, cmy);
}

// 0 when the kernel takes the record; the reason it does not otherwise (the record then leaves its macroblock untouched)
__device__ __forceinline__ int mpv_mc_reject(const MpvMcPic &P, const FFMpvMCRecord &r)
{
    if (r.mb_x >= P.mb_w || r.mb_y >= P.mb_rows || r.mv_dir > 7 || r.mv_type > MPV_MC_DMV) return 1;
    const bool frame = P.structure == MPV_PICT_FRAME;
    if (P.h263) {
        if (r.mv_type != MPV_MC_16X16 && r.mv_type != MPV_MC_8X8) return 2;
    } else {
        if (r.mv_type == MPV_MC_8X8 || (frame && r.mv_type == MPV_MC_16X8) || (!frame && r.mv_type == MPV_MC_16X16)) return 2;
    }
    for (int dir = 0; dir < 2; dir++)
        if ((r.mv_dir >> dir) & 1)
            if (!P.ref[dir][0] || !P.ref[dir][1] || !P.ref[dir][2]) return 3;
    return 0;
}

// mpv_mc_reject for a picture of kind IL: an interlaced H.263-family picture also takes FIELD records (the other checks hold for them)
template <int IL>
__device__ __forceinline__ int mpv_mc_reject_kind(const MpvMcPic &P, const FFMpvMCRecord &r)
{
    if (IL && P.h263 && r.mv_type == MPV_MC_FIELD) {
        FFMpvMCRecord q = r;
        q.mv_type = MPV_MC_16X16;
        return mpv_mc_reject(P, q);
    }
    return mpv_mc_reject(P, r);
}

// ff_mpv_motion for every direction of the record, in ff_mpv_reconstruct_mb's order; column m of the lane map only
template <int CF, int IL>
__device__ __forceinline__ void mpv_mc_column(const MpvMcPic &P, const FFMpvMCRecord &r, int m)
{
    MpvLane L;
    if (CF == 1) {
        L.pl = m < 16 ? 0 : 1 + ((m - 16) >> 3);
        L.c = L.pl ? (m & 7) : m;
        const int bs = L.pl ? 8 : 16;
        L.dls = (ptrdiff_t)P.pic_k * P.ls[L.pl != 0];
        L.dcol = P.dest[L.pl] + (ptrdiff_t)r.mb_y * bs * L.dls + r.mb_x * bs + L.c;
    } else {               // the chroma block of a macroblock: 8 x 16 in 4:2:2, 16 x 16 in 4:4:4
        L.pl = CF == 3 ? m >> 4 : m < 16 ? 0 : 1 + ((m - 16) >> 3);
        L.c = CF == 3 ? m & 15 : L.pl ? (m & 7) : m;
        const int bw = L.pl && CF == 2 ? 8 : 16;
        L.dls = (ptrdiff_t)P.pic_k * P.ls[L.pl != 0];
        L.dcol = P.dest[L.pl] + (ptrdiff_t)r.mb_y * 16 * L.dls + r.mb_x * bw + L.c;
    }
    const bool frame = P.structure == MPV_PICT_FRAME, second_p = !P.b_pic && !P.first_field;
    int avg = 0;
    for (int dir = 0; dir < 2; dir++) {
        if (!((r.mv_dir >> dir) & 1)) continue;
        const uint8_t *const *ref = P.ref[dir];
        const int no_rnd = !avg && P.no_rnd && !P.b_pic;
        const int16_t (*mv)[2] = r.mv[dir];
        const uint8_t *fs = r.field_select[dir];
        switch (r.mv_type) {
        case MPV_MC_16X16:
            if (P.h263 && P.qpel) mpv_qpel_motion(P, L, r, ref, no_rnd, avg, mv[0][0], mv[0][1]);
            else mpv_mpeg_motion<CF, IL>(P, L, r, 0, 0, 0, ref, no_rnd, avg, mv[0][0], mv[0][1], 16, r.mb_y, 0);
            break;
        case MPV_MC_8X8:
            mpv_apply_8x8(P, L, r, dir, ref, no_rnd, avg);
            break;
        case MPV_MC_FIELD:
            if (frame && IL && P.qpel) {
                for (int i = 0; i < 2; i++) mpv_qpel_field(P, L, r, i, fs[i], ref, no_rnd, avg, mv[i][0], mv[i][1]);
            } else if (frame) {
                mpv_mpeg_motion<CF, IL>(P, L, r, 1, 0, fs[0], ref, no_rnd, avg, mv[0][0], mv[0][1], 8, r.mb_y, 0);
                mpv_mpeg_motion<CF, IL>(P, L, r, 1, 1, fs[1], ref, no_rnd, avg, mv[1][0], mv[1][1], 8, r.mb_y, 0);
            } else {
                const uint8_t *const *rp = (P.structure != fs[0] + 1 && second_p) ? P.cur : ref;
                mpv_mpeg_motion<CF, IL>(P, L, r, 0, 0, fs[0], rp, no_rnd, avg, mv[0][0], mv[0][1], 16, r.mb_y, 0);
            }
            break;
        case MPV_MC_16X8:      // field pictures: the lower half starts 16 frame lines = 8 field lines down
            for (int i = 0; i < 2; i++) {
                const uint8_t *const *rp = (P.structure == fs[i] + 1 || !second_p) ? ref : P.cur;
                mpv_mpeg_motion<CF, IL>(P, L, r, 0, 0, fs[i], rp, no_rnd, avg, mv[i][0], mv[i][1] + 16 * i, 8, r.mb_y, 8 * i);
            }
            break;
        case MPV_MC_DMV:       // put then avg between the two parities, inside one direction
            if (frame) {
                for (int i = 0; i < 2; i++) {
                    for (int j = 0; j < 2; j++)
                        mpv_mpeg_motion<CF, IL>(P, L, r, 1, j, j ^ i, ref, i ? 0 : no_rnd, i ? 1 : avg, mv[2 * i + j][0], mv[2 * i + j][1], 8, r.mb_y, 0);
                }
            } else {
                const uint8_t *const *rp = ref;
                for (int i = 0; i < 2; i++) {
                    mpv_mpeg_motion<CF, IL>(P, L, r, 0, 0, P.structure != i + 1, rp, i ? 0 : no_rnd, i ? 1 : avg, mv[2 * i][0], mv[2 * i][1], 16, r.mb_y, 0);
                    if (!P.first_field) rp = P.cur;            // the opposite parity of a second field is in the same frame
                }
            }
            break;
        }
        avg = 1;
    }
}

// the lane's columns of the record: one of the 16 + 8 + 8 map, or columns lane and lane + 32 of 4:4:4's 16 + 16 + 16
template <int CF = 1, int IL = 0>
__device__ __forceinline__ void mpv_mc_lane(const MpvMcPic &P, const FFMpvMCRecord &r, int lane)
{
    if (CF == 3) {
        for (int m = lane; m < 48; m += 32) mpv_mc_column<CF, IL>(P, r, m);
    } else {
        mpv_mc_column<CF, IL>(P, r, lane);
    }
}

}  // namespace avb
