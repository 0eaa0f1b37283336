/*
 * oracle/port/orc_mpvmc.c -- TEST INFRASTRUCTURE, NOT PRODUCT.
 *
 * CPU restatement (plain C) of the motion compensation of the mpegvideo decoders, ff_mpv_motion() (libavcodec/mpegvideo_motion.c:192-968)
 * as ff_mpv_reconstruct_mb() drives it (mpegvideo.c:1548-1578), for the cases include/avdsp_b200.h lists: MPEG-1 / MPEG-2 16X16, FIELD,
 * 16X8 and DMV in frame and field pictures; H.263 / MPEG-4 16X16 and 8X8, half- and quarter-sample.  Whole-block operations on pointers,
 * as the C library calls them: an emulated edge is a real copy of the clamped block into a scratch buffer, the half-sample ops are the
 * rounded / truncated means of hpeldsp, the quarter-sample ops build the full-sample, horizontal and vertical planes of qpeldsp.
 * Same arguments as ref_mpvmc_picture (oracle/refbuild/refapi_mpvmc.c); pinned picture for picture against it by tests/test_mpv_mc_cpu.py.
 */
#include <stdint.h>
#include <stddef.h>
#include <string.h>

typedef struct Rec {
    uint16_t mb_x, mb_y;
    uint8_t mv_dir, mv_type, field_select[2][2];
    int16_t mv[2][4][2];
    uint8_t pad[2];
} Rec;

enum { T16X16, T8X8, T16X8, TFIELD, TDMV };
enum { PUT, PUT_NO_RND, AVG };

typedef struct Ctx {
    int ls, uvls, pic_ls, pic_uvls, width, height, h_edge, v_edge, h263, structure, first_field, b, no_rnd, qpel, bugs;
    int mb_x, mb_y;
    uint8_t **cur;
    uint8_t emu[3][32 * 32];      /* edge emulation buffers (stride 32), one per plane */
} Ctx;

static int imax(int a, int b) { return a > b ? a : b; }
static int iclip(int v, int lo, int hi) { return v < lo ? lo : v > hi ? hi : v; }
static uint8_t clip8(int v) { return v < 0 ? 0 : v > 255 ? 255 : (uint8_t)v; }

/* videodsp emulated_edge_mc: the bw x bh block at (sx, sy) of a w x h picture, samples outside replaced by the nearest edge sample */
static const uint8_t *emulate(uint8_t *buf, const uint8_t *plane, ptrdiff_t stride, int bw, int bh, int sx, int sy, int w, int h)
{
    for (int y = 0; y < bh; y++)
        for (int x = 0; x < bw; x++)
            buf[y * 32 + x] = plane[(ptrdiff_t)iclip(sy + y, 0, h - 1) * stride + iclip(sx + x, 0, w - 1)];
    return buf;
}

static void store(uint8_t *d, int v, int op) { *d = op == AVG ? (uint8_t)((*d + v + 1) >> 1) : (uint8_t)v; }

/* hpeldsp put / put_no_rnd / avg pixels, w wide, h rows, at half-sample position dxy */
static void hpel(uint8_t *dst, ptrdiff_t ds, const uint8_t *src, ptrdiff_t ss, int w, int h, int dxy, int op)
{
    const int nr = op == PUT_NO_RND;
    for (int y = 0; y < h; y++)
        for (int x = 0; x < w; x++) {
            const uint8_t *p = src + y * ss + x;
            int v;
            switch (dxy) {
            case 0: v = p[0]; break;
            case 1: v = (p[0] + p[1] + 1 - nr) >> 1; break;
            case 2: v = (p[0] + p[ss] + 1 - nr) >> 1; break;
            default: v = (p[0] + p[1] + p[ss] + p[ss + 1] + 2 - nr) >> 2; break;
            }
            store(dst + y * ds + x, v, op);
        }
}

/* the MPEG-4 8-tap lowpass over an n-sample line s[0..n], mirrored at both ends */
static int lowpass(const int *s, int n, int i, int rnd)
{
#define S(j) s[(j) < 0 ? -1 - (j) : (j) > n ? 2 * n + 1 - (j) : (j)]
    const int v = 20 * (S(i) + S(i + 1)) - 6 * (S(i - 1) + S(i + 2)) + 3 * (S(i - 2) + S(i + 3)) - (S(i - 3) + S(i + 4));
#undef S
    return clip8((v + rnd) >> 5);
}

/* qpeldsp put / put_no_rnd / avg qpel pixels, n x n, quarter-sample position mc = x + 4 * y */
static void qpel(uint8_t *dst, ptrdiff_t ds, const uint8_t *src, ptrdiff_t ss, int n, int mc, int op)
{
    const int qx = mc & 3, qy = mc >> 2, nr = op == PUT_NO_RND, rnd = nr ? 15 : 16, up = !nr;
    const int rows = qy ? n + 1 : n, cols = qx ? n + 1 : n;
    int full[17][17], half[17][17], line[17], col[17];
    for (int y = 0; y < rows; y++)
        for (int x = 0; x < cols; x++) full[y][x] = src[y * ss + x];
    for (int y = 0; y < rows; y++) {
        for (int x = 0; x < cols; x++) line[x] = full[y][x];
        for (int x = 0; x < n; x++) {
            if (!qx) { half[y][x] = full[y][x]; continue; }
            const int h = lowpass(line, n, x, rnd);
            half[y][x] = qx == 2 ? h : (full[y][x + (qx == 3)] + h + up) >> 1;
        }
    }
    for (int x = 0; x < n; x++) {
        for (int y = 0; y < rows; y++) col[y] = half[y][x];
        for (int y = 0; y < n; y++) {
            int v = half[y][x];
            if (qy) {
                const int l = lowpass(col, n, y, rnd);
                v = qy == 2 ? l : (half[y + (qy == 3)][x] + l + up) >> 1;
            }
            store(dst + y * ds + x, v, op);
        }
    }
}

/* mpeg_motion_internal (4:2:0) */
static void mpeg_motion(Ctx *c, uint8_t **dest, int fb, int bottom, int fs, uint8_t **ref, int op, int mx, int my, int h, int mb_y)
{
    const int v_edge = c->v_edge >> fb;
    const ptrdiff_t ls = (ptrdiff_t)c->pic_ls << fb, uvls = (ptrdiff_t)c->pic_uvls << fb;
    const int dxy = ((my & 1) << 1) | (mx & 1);
    const int sx = c->mb_x * 16 + (mx >> 1), sy = (mb_y << (4 - fb)) + (my >> 1);
    int uvdxy, ux, uy;
    if (c->h263) {
        uvdxy = dxy | (my & 2) | ((mx & 2) >> 1);
        ux = sx >> 1;
        uy = sy >> 1;
    } else {
        const int cx = mx / 2, cy = my / 2;
        uvdxy = ((cy & 1) << 1) | (cx & 1);
        ux = c->mb_x * 8 + (cx >> 1);
        uy = (mb_y << (3 - fb)) + (cy >> 1);
    }
    const uint8_t *py, *pu, *pv;
    ptrdiff_t sls = ls, suvls = uvls;
    if ((unsigned)sx > (unsigned)imax(c->h_edge - (mx & 1) - 16, 0) || (unsigned)sy > (unsigned)imax(v_edge - (my & 1) - h, 0)) {
        if (!c->h263) return;
        /* frame pictures only here (field MC of the H.263 family is not covered): 17x17 luma, 9x9 chroma */
        py = emulate(c->emu[0], ref[0], c->ls, 17, 17, sx, sy, c->h_edge, c->v_edge);
        pu = emulate(c->emu[1], ref[1], c->uvls, 9, 9, ux, uy, c->h_edge >> 1, c->v_edge >> 1);
        pv = emulate(c->emu[2], ref[2], c->uvls, 9, 9, ux, uy, c->h_edge >> 1, c->v_edge >> 1);
        sls = suvls = 32;
        hpel(dest[0], ls, py, sls, 16, h, dxy, op);
        hpel(dest[1], uvls, pu, suvls, 8, h >> 1, uvdxy, op);
        hpel(dest[2], uvls, pv, suvls, 8, h >> 1, uvdxy, op);
        return;
    }
    py = ref[0] + sy * ls + sx + (fs ? c->ls : 0);
    pu = ref[1] + uy * uvls + ux + (fs ? c->uvls : 0);
    pv = ref[2] + uy * uvls + ux + (fs ? c->uvls : 0);
    const ptrdiff_t dy = bottom ? c->ls : 0, duv = bottom ? c->uvls : 0;
    hpel(dest[0] + dy, ls, py, ls, 16, h, dxy, op);
    hpel(dest[1] + duv, uvls, pu, uvls, 8, h >> 1, uvdxy, op);
    hpel(dest[2] + duv, uvls, pv, uvls, 8, h >> 1, uvdxy, op);
}

/* qpel_motion, frame-based */
static void qpel_motion(Ctx *c, uint8_t **dest, uint8_t **ref, int op, int mx, int my)
{
    const int dxy = ((my & 3) << 2) | (mx & 3);
    const int sx = c->mb_x * 16 + (mx >> 2), sy = c->mb_y * 16 + (my >> 2);
    static const int rtab[8] = { 0, 0, 1, 1, 0, 0, 0, 1 };
    int cx, cy;
    if (c->bugs & 256) {
        cx = (mx >> 1) + rtab[mx & 7];
        cy = (my >> 1) + rtab[my & 7];
    } else if (c->bugs & 64) {
        cx = (mx >> 1) | (mx & 1);
        cy = (my >> 1) | (my & 1);
    } else {
        cx = mx / 2;
        cy = my / 2;
    }
    cx = (cx >> 1) | (cx & 1);
    cy = (cy >> 1) | (cy & 1);
    const int uvdxy = (cx & 1) | ((cy & 1) << 1);
    const int ux = c->mb_x * 8 + (cx >> 1), uy = c->mb_y * 8 + (cy >> 1);
    const uint8_t *py = ref[0] + sy * c->ls + sx, *pu = ref[1] + uy * c->uvls + ux, *pv = ref[2] + uy * c->uvls + ux;
    ptrdiff_t sls = c->ls, suvls = c->uvls;
    if ((unsigned)sx > (unsigned)imax(c->h_edge - (mx & 3) - 16, 0) || (unsigned)sy > (unsigned)imax(c->v_edge - (my & 3) - 16, 0)) {
        py = emulate(c->emu[0], ref[0], c->ls, 17, 17, sx, sy, c->h_edge, c->v_edge);
        pu = emulate(c->emu[1], ref[1], c->uvls, 9, 9, ux, uy, c->h_edge >> 1, c->v_edge >> 1);
        pv = emulate(c->emu[2], ref[2], c->uvls, 9, 9, ux, uy, c->h_edge >> 1, c->v_edge >> 1);
        sls = suvls = 32;
    }
    qpel(dest[0], c->ls, py, sls, 16, dxy, op);
    hpel(dest[1], c->uvls, pu, suvls, 8, 8, uvdxy, op);
    hpel(dest[2], c->uvls, pv, suvls, 8, 8, uvdxy, op);
}

/* chroma_4mv_motion */
static void chroma_4mv(Ctx *c, uint8_t **dest, uint8_t **ref, int op, int mx, int my)
{
    static const uint8_t tab[16] = { 0, 0, 0, 1, 1, 1, 1, 1, 0, 0, 0, 0, 0, 0, 1, 1 };
    mx = tab[mx & 15] + (mx >> 3);
    my = tab[my & 15] + (my >> 3);
    int dxy = ((my & 1) << 1) | (mx & 1);
    int sx = iclip(c->mb_x * 8 + (mx >> 1), -8, c->width >> 1), sy = iclip(c->mb_y * 8 + (my >> 1), -8, c->height >> 1);
    if (sx == c->width >> 1) dxy &= ~1;
    if (sy == c->height >> 1) dxy &= ~2;
    const int emu = (unsigned)sx > (unsigned)imax((c->h_edge >> 1) - (dxy & 1) - 8, 0) ||
                    (unsigned)sy > (unsigned)imax((c->v_edge >> 1) - (dxy >> 1) - 8, 0);
    for (int p = 1; p < 3; p++) {
        const uint8_t *s = ref[p] + sy * c->uvls + sx;
        ptrdiff_t ss = c->uvls;
        if (emu) { s = emulate(c->emu[p], ref[p], c->uvls, 9, 9, sx, sy, c->h_edge >> 1, c->v_edge >> 1); ss = 32; }
        hpel(dest[p], c->uvls, s, ss, 8, 8, dxy, op);
    }
}

/* apply_8x8: hpel_motion / the quarter-sample loop for the four luma blocks, then chroma_4mv_motion */
static void apply_8x8(Ctx *c, uint8_t **dest, const Rec *r, int dir, uint8_t **ref, int op)
{
    int smx = 0, smy = 0;
    for (int i = 0; i < 4; i++) {
        const int mx = r->mv[dir][i][0], my = r->mv[dir][i][1];
        int dxy, sx, sy, emu;
        if (c->qpel) {
            dxy = ((my & 3) << 2) | (mx & 3);
            sx = iclip(c->mb_x * 16 + (mx >> 2) + (i & 1) * 8, -16, c->width);
            if (sx == c->width) dxy &= ~3;
            sy = iclip(c->mb_y * 16 + (my >> 2) + (i >> 1) * 8, -16, c->height);
            if (sy == c->height) dxy &= ~12;
            emu = (unsigned)sx > (unsigned)imax(c->h_edge - (mx & 3) - 8, 0) || (unsigned)sy > (unsigned)imax(c->v_edge - (my & 3) - 8, 0);
            smx += mx / 2;
            smy += my / 2;
        } else {
            dxy = 0;
            sx = iclip(c->mb_x * 16 + (i & 1) * 8 + (mx >> 1), -16, c->width);
            if (sx != c->width) dxy |= mx & 1;
            sy = iclip(c->mb_y * 16 + (i >> 1) * 8 + (my >> 1), -16, c->height);
            if (sy != c->height) dxy |= (my & 1) << 1;
            emu = (unsigned)sx > (unsigned)imax(c->h_edge - (mx & 1) - 8, 0) || (unsigned)sy > (unsigned)imax(c->v_edge - (my & 1) - 8, 0);
            smx += mx;
            smy += my;
        }
        const uint8_t *s = ref[0] + sy * c->ls + sx;
        ptrdiff_t ss = c->ls;
        if (emu) { s = emulate(c->emu[0], ref[0], c->ls, 9, 9, sx, sy, c->h_edge, c->v_edge); ss = 32; }
        uint8_t *d = dest[0] + (i & 1) * 8 + (i >> 1) * 8 * c->ls;
        if (c->qpel) qpel(d, c->ls, s, ss, 8, dxy, op);
        else         hpel(d, c->ls, s, ss, 8, 8, dxy, op);
    }
    chroma_4mv(c, dest, ref, op, smx, smy);
}

/* ff_mpv_motion for one direction */
static void motion(Ctx *c, uint8_t **dest, const Rec *r, int dir, uint8_t **ref, int op, int mb_y)
{
    const int frame = c->structure == 3, second_p = !c->b && !c->first_field;
    const int16_t (*mv)[2] = r->mv[dir];
    const uint8_t *fs = r->field_select[dir];
    switch (r->mv_type) {
    case T16X16:
        if (c->h263 && c->qpel) qpel_motion(c, dest, ref, op, mv[0][0], mv[0][1]);
        else mpeg_motion(c, dest, 0, 0, 0, ref, op, mv[0][0], mv[0][1], 16, mb_y);
        break;
    case T8X8:
        apply_8x8(c, dest, r, dir, ref, op);
        break;
    case TFIELD:
        if (frame) {
            mpeg_motion(c, dest, 1, 0, fs[0], ref, op, mv[0][0], mv[0][1], 8, mb_y);
            mpeg_motion(c, dest, 1, 1, fs[1], ref, op, mv[1][0], mv[1][1], 8, mb_y);
        } else {
            mpeg_motion(c, dest, 0, 0, fs[0], (c->structure != fs[0] + 1 && second_p) ? c->cur : ref, op, mv[0][0], mv[0][1], 16, mb_y);
        }
        break;
    case T16X8: {
        uint8_t *d[3] = { dest[0], dest[1], dest[2] };
        for (int i = 0; i < 2; i++) {
            mpeg_motion(c, d, 0, 0, fs[i], (c->structure == fs[i] + 1 || !second_p) ? ref : c->cur, op, mv[i][0], mv[i][1] + 16 * i, 8, mb_y);
            d[0] += 16 * c->ls;
            d[1] += 8 * c->uvls;
            d[2] += 8 * c->uvls;
        }
        break;
    }
    case TDMV:
        if (frame) {
            for (int i = 0; i < 2; i++) {
                for (int j = 0; j < 2; j++)
                    mpeg_motion(c, dest, 1, j, j ^ i, ref, op, mv[2 * i + j][0], mv[2 * i + j][1], 8, mb_y);
                op = AVG;
            }
        } else {
            for (int i = 0; i < 2; i++) {
                mpeg_motion(c, dest, 0, 0, c->structure != i + 1, ref, op, mv[2 * i][0], mv[2 * i][1], 16, mb_y);
                op = AVG;
                if (!c->first_field) ref = c->cur;
            }
        }
        break;
    }
}

int orc_mpvmc_picture(uint8_t **dest, uint8_t **cur, uint8_t **last, uint8_t **next, const int *prm, const Rec *recs, size_t n)
{
    Ctx c;
    memset(&c, 0, sizeof(c));
    c.ls = prm[0]; c.uvls = prm[1]; c.pic_ls = prm[2]; c.pic_uvls = prm[3];
    c.width = prm[6]; c.height = prm[7]; c.h_edge = prm[8]; c.v_edge = prm[9];
    c.h263 = prm[10] == 2; c.structure = prm[11]; c.first_field = prm[12]; c.b = prm[13]; c.no_rnd = prm[14];
    c.qpel = c.h263 && prm[15]; c.bugs = prm[16];
    c.cur = cur;
    for (size_t i = 0; i < n; i++) {
        const Rec *r = &recs[i];
        c.mb_x = r->mb_x;
        c.mb_y = r->mb_y;                 /* the row in the picture: what mpeg_motion receives (mb_y, or s->mb_y >> 1 in a field) */
        uint8_t *d[3] = { dest[0] + (ptrdiff_t)r->mb_y * 16 * c.pic_ls + r->mb_x * 16,
                          dest[1] + (ptrdiff_t)r->mb_y * 8 * c.pic_uvls + r->mb_x * 8,
                          dest[2] + (ptrdiff_t)r->mb_y * 8 * c.pic_uvls + r->mb_x * 8 };
        int op = (c.no_rnd && !c.b) ? PUT_NO_RND : PUT;
        if (r->mv_dir & 1) { motion(&c, d, r, 0, last, op, r->mb_y); op = AVG; }
        if (r->mv_dir & 2) motion(&c, d, r, 1, next, op, r->mb_y);
    }
    return 0;
}
