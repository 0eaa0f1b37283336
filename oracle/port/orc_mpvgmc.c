/*
 * oracle/port/orc_mpvgmc.c -- TEST INFRASTRUCTURE, NOT PRODUCT.
 *
 * CPU restatement (plain C) of MPEG-4 global motion compensation in an S-VOP: what ff_mpv_motion (libavcodec/mpegvideo_motion.c:834-843)
 * does for a 16X16 macroblock with s->mcsel set -- gmc1_motion (:37-132) when real_sprite_warping_points is 1, gmc_motion (:134-190)
 * otherwise -- with MpegVideoDSPContext's gmc1_c and ff_gmc_c (libavcodec/mpegvideodsp.c:24-108) written formula by formula.  Every other
 * record goes through orc_mpvmc_picture (orc_mpvmc.c).  Emulated edges are read with clamped coordinates, which is what
 * emulated_edge_mc's buffer holds.  Same arguments as ref_mpvmc_gmc_picture (oracle/refbuild/refapi_mpvgmc.c); pinned to the reference
 * by tests/test_mpv_gmc_cpu.py.
 */
#include <stdint.h>
#include <stddef.h>

typedef struct Rec {
    uint16_t mb_x, mb_y;
    uint8_t mv_dir, mv_type, field_select[2][2];
    int16_t mv[2][4][2];
    uint8_t mcsel, pad;
} Rec;

int orc_mpvmc_picture(uint8_t **dest, uint8_t **cur, uint8_t **last, uint8_t **next, const int *prm, const Rec *recs, size_t n);

static int imax(int a, int b) { return a > b ? a : b; }
static int iclip(int v, int lo, int hi) { return v < lo ? lo : v > hi ? hi : v; }

/* sample (x, y) of a plane, clamped to [0, w) x [0, h) when emu is set (the edge emulation buffer), else read directly */
static int px(const uint8_t *p, ptrdiff_t ls, int x, int y, int emu, int w, int h)
{
    if (emu) { x = iclip(x, 0, w - 1); y = iclip(y, 0, h - 1); }
    return p[(ptrdiff_t)y * ls + x];
}

/* gmc1_c (mpegvideodsp.c:24-45) on a bw x bw block at (sx, sy) */
static void gmc1(uint8_t *dst, ptrdiff_t ls, const uint8_t *p, int sx, int sy, int emu, int w, int h, int bw, int x16, int y16, int rounder)
{
    const int A = (16 - x16) * (16 - y16), B = x16 * (16 - y16), C = (16 - x16) * y16, D = x16 * y16;
    for (int y = 0; y < bw; y++)
        for (int x = 0; x < bw; x++)
            dst[y * ls + x] = (uint8_t)((A * px(p, ls, sx + x, sy + y, emu, w, h) + B * px(p, ls, sx + x + 1, sy + y, emu, w, h) +
                                         C * px(p, ls, sx + x, sy + y + 1, emu, w, h) + D * px(p, ls, sx + x + 1, sy + y + 1, emu, w, h) +
                                         rounder) >> 8);
}

/* ff_gmc_c (mpegvideodsp.c:47-108), 8 columns, h rows; running sums as in C (-fwrapv) */
static void gmc(uint8_t *dst, const uint8_t *src, int stride, int h, int ox, int oy, int dxx, int dxy, int dyx, int dyy, int shift, int r,
                int width, int height)
{
    const int s = 1 << shift;
    width--;
    height--;
    for (int y = 0; y < h; y++) {
        int vx = ox, vy = oy;
        for (int x = 0; x < 8; x++) {
            int src_x = vx >> 16, src_y = vy >> 16;
            const int fx = src_x & (s - 1), fy = src_y & (s - 1);
            src_x >>= shift;
            src_y >>= shift;
            int v;
            if ((unsigned)src_x < (unsigned)width && (unsigned)src_y < (unsigned)height) {
                const uint8_t *q = src + src_x + (ptrdiff_t)src_y * stride;
                v = ((q[0] * (s - fx) + q[1] * fx) * (s - fy) + (q[stride] * (s - fx) + q[stride + 1] * fx) * fy + r) >> (shift * 2);
            } else if ((unsigned)src_x < (unsigned)width) {
                const uint8_t *q = src + src_x + (ptrdiff_t)iclip(src_y, 0, height) * stride;
                v = ((q[0] * (s - fx) + q[1] * fx) * s + r) >> (shift * 2);
            } else if ((unsigned)src_y < (unsigned)height) {
                const uint8_t *q = src + iclip(src_x, 0, width) + (ptrdiff_t)src_y * stride;
                v = ((q[0] * (s - fy) + q[stride] * fy) * s + r) >> (shift * 2);
            } else {
                v = src[iclip(src_x, 0, width) + (ptrdiff_t)iclip(src_y, 0, height) * stride];
            }
            dst[y * stride + x] = (uint8_t)v;
            vx += dxx;
            vy += dyx;
        }
        ox += dxy;
        oy += dyy;
    }
}

/* the C slots, for the slot tests where _ref was not built */
void orc_gmc1(uint8_t *dst, uint8_t *src, int stride, int h, int x16, int y16, int rounder)
{
    const int A = (16 - x16) * (16 - y16), B = x16 * (16 - y16), C = (16 - x16) * y16, D = x16 * y16;
    for (int y = 0; y < h; y++)
        for (int x = 0; x < 8; x++) {
            const uint8_t *q = src + (ptrdiff_t)y * stride + x;
            dst[(ptrdiff_t)y * stride + x] = (uint8_t)((A * q[0] + B * q[1] + C * q[stride] + D * q[stride + 1] + rounder) >> 8);
        }
}

void orc_gmc(uint8_t *dst, uint8_t *src, int stride, int h, int ox, int oy, int dxx, int dxy, int dyx, int dyy, int shift, int r, int width,
             int height)
{
    gmc(dst, src, stride, h, ox, oy, dxx, dxy, dyx, dyy, shift, r, width, height);
}

/* hpeldsp put / put_no_rnd pixels16 (the integer / half-sample fall-back of gmc1_motion, :79-87) */
static void put16(uint8_t *dst, ptrdiff_t ls, const uint8_t *p, int sx, int sy, int emu, int w, int h, int dxy, int nr)
{
    for (int y = 0; y < 16; y++)
        for (int x = 0; x < 16; x++) {
            const int a = px(p, ls, sx + x, sy + y, emu, w, h), b = px(p, ls, sx + x + 1, sy + y, emu, w, h);
            const int c = px(p, ls, sx + x, sy + y + 1, emu, w, h), d = px(p, ls, sx + x + 1, sy + y + 1, emu, w, h);
            dst[y * ls + x] = (uint8_t)(dxy == 0 ? a : dxy == 1 ? (a + b + 1 - nr) >> 1 : dxy == 2 ? (a + c + 1 - nr) >> 1 : (a + b + c + d + 2 - nr) >> 2);
        }
}

/* gmc1_motion (:37-132) */
static void gmc1_motion(uint8_t **dest, uint8_t **ref, const int *prm, const int *sp, int mb_x, int mb_y)
{
    const int ls = prm[0], uvls = prm[1], width = prm[6], height = prm[7], he = prm[8], ve = prm[9], nr = prm[14], a = sp[0];
    int mx = sp[2], my = sp[3];
    int sx = mb_x * 16 + (mx >> (a + 1)), sy = mb_y * 16 + (my >> (a + 1));
    mx = (int)((unsigned)mx << (3 - a));
    my = (int)((unsigned)my << (3 - a));
    sx = iclip(sx, -16, width);                            /* :52-57: clipped to width / height, fraction dropped at the far end */
    if (sx == width) mx = 0;
    sy = iclip(sy, -16, height);
    if (sy == height) my = 0;
    int emu = (unsigned)sx >= (unsigned)imax(he - 17, 0) || (unsigned)sy >= (unsigned)imax(ve - 17, 0);     /* :64-65, 17 x 17 */
    uint8_t *dy = dest[0] + (ptrdiff_t)mb_y * 16 * ls + mb_x * 16;
    if ((mx | my) & 7)
        gmc1(dy, ls, ref[0], sx, sy, emu, he, ve, 16, mx & 15, my & 15, 128 - nr);
    else
        put16(dy, ls, ref[0], sx, sy, emu, he, ve, ((mx >> 3) & 1) | ((my >> 2) & 2), nr);
    mx = sp[4];
    my = sp[5];
    sx = mb_x * 8 + (mx >> (a + 1));
    sy = mb_y * 8 + (my >> (a + 1));
    mx = (int)((unsigned)mx << (3 - a));
    my = (int)((unsigned)my << (3 - a));
    sx = iclip(sx, -8, width >> 1);
    if (sx == width >> 1) mx = 0;
    sy = iclip(sy, -8, height >> 1);
    if (sy == height >> 1) my = 0;
    emu = (unsigned)sx >= (unsigned)imax((he >> 1) - 9, 0) || (unsigned)sy >= (unsigned)imax((ve >> 1) - 9, 0);     /* :108-109, 9 x 9 */
    for (int p = 1; p < 3; p++)
        gmc1(dest[p] + (ptrdiff_t)mb_y * 8 * uvls + mb_x * 8, uvls, ref[p], sx, sy, emu, he >> 1, ve >> 1, 8, mx & 15, my & 15, 128 - nr);
}

/* gmc_motion (:134-190): two 8-wide luma calls and one per chroma plane */
static void gmc_motion(uint8_t **dest, uint8_t **ref, const int *prm, const int *sp, int mb_x, int mb_y)
{
    const int ls = prm[0], uvls = prm[1], he = prm[8], ve = prm[9], nr = prm[14], a = sp[0];
    const int *off = sp + 2, *d = sp + 6;                  /* sprite_offset[2][2], sprite_delta[2][2] */
    const int shift = a + 1, r = (1 << (2 * a + 1)) - nr;
    uint8_t *dy = dest[0] + (ptrdiff_t)mb_y * 16 * ls + mb_x * 16;
    int ox = off[0] + d[0] * mb_x * 16 + d[1] * mb_y * 16, oy = off[1] + d[2] * mb_x * 16 + d[3] * mb_y * 16;
    gmc(dy, ref[0], ls, 16, ox, oy, d[0], d[1], d[2], d[3], shift, r, he, ve);
    gmc(dy + 8, ref[0], ls, 16, ox + d[0] * 8, oy + d[2] * 8, d[0], d[1], d[2], d[3], shift, r, he, ve);
    ox = off[2] + d[0] * mb_x * 8 + d[1] * mb_y * 8;
    oy = off[3] + d[2] * mb_x * 8 + d[3] * mb_y * 8;
    for (int p = 1; p < 3; p++)
        gmc(dest[p] + (ptrdiff_t)mb_y * 8 * uvls + mb_x * 8, ref[p], uvls, 8, ox, oy, d[0], d[1], d[2], d[3], shift, r, he >> 1, ve >> 1);
}

/* sprite: sprite_warping_accuracy, real_sprite_warping_points, sprite_offset[2][2], sprite_delta[2][2] */
int orc_mpvgmc_picture(uint8_t **dest, uint8_t **cur, uint8_t **last, uint8_t **next, const int *prm, const Rec *recs, size_t n,
                       const int *sprite)
{
    for (size_t k = 0; k < n; k++) {
        const Rec *r = &recs[k];
        if (r->mv_type != 0 || !r->mcsel) {
            orc_mpvmc_picture(dest, cur, last, next, prm, r, 1);
            continue;
        }
        for (int dir = 0; dir < 2; dir++) {                /* gmc1 / gmc put for every direction ff_mpv_reconstruct_mb runs */
            if (!((r->mv_dir >> dir) & 1)) continue;
            if (sprite[1] == 1) gmc1_motion(dest, dir ? next : last, prm, sprite, r->mb_x, r->mb_y);
            else                gmc_motion(dest, dir ? next : last, prm, sprite, r->mb_x, r->mb_y);
        }
    }
    return 0;
}
