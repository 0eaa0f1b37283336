/*
 * oracle/port/orc_mpvobmc.c -- TEST INFRASTRUCTURE, NOT PRODUCT.
 *
 * CPU restatement (plain C) of H.263 overlapped block motion compensation, apply_obmc (libavcodec/mpegvideo_motion.c:403-728), over the
 * records' FFMpvOBMCRecord copies of what it reads: the neighbour substitutions of :674-700, five hpel_motion predictions per 8x8 luma
 * block combined with put_obmc's weights, chroma_4mv_motion with the sum of the own vectors.  Whole-block operations on buffers like the
 * C code; emulated edges are copied into a buffer.  Same arguments as ref_mpvobmc_picture (oracle/refbuild/refapi_mpvobmc.c); B pictures
 * ignore obmc and go through orc_mpvmc_picture.  Pinned to the reference by tests/test_mpv_obmc_cpu.py.
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

typedef struct ObmcRec {
    int16_t mv[4][2], top[2][2], left[2][2], right[2][2];
    uint32_t mb_type_top, mb_type_left, mb_type_right;
} ObmcRec;

int orc_mpvmc_picture(uint8_t **dest, uint8_t **cur, uint8_t **last, uint8_t **next, const int *prm, const Rec *recs, size_t n);

typedef struct Ctx { int ls, uvls, width, height, h_edge, v_edge, no_rnd; } Ctx;

static int imax(int a, int b) { return a > b ? a : b; }
static int iclip(int v, int lo, int hi) { return v < lo ? lo : v > hi ? hi : v; }

/* videodsp emulated_edge_mc into a 9 x 9 buffer of stride 16 */
static const uint8_t *emulate(uint8_t *buf, const uint8_t *plane, ptrdiff_t stride, int sx, int sy, int w, int h)
{
    for (int y = 0; y < 9; y++)
        for (int x = 0; x < 9; x++) buf[y * 16 + x] = plane[(ptrdiff_t)iclip(sy + y, 0, h - 1) * stride + iclip(sx + x, 0, w - 1)];
    return buf;
}

/* hpeldsp put / put_no_rnd pixels8 */
static void put8(uint8_t *dst, ptrdiff_t ds, const uint8_t *p, ptrdiff_t ss, int dxy, int nr)
{
    for (int y = 0; y < 8; y++)
        for (int x = 0; x < 8; x++) {
            const uint8_t *s = p + y * ss + x;
            dst[y * ds + x] = (uint8_t)(dxy == 0 ? s[0] : dxy == 1 ? (s[0] + s[1] + 1 - nr) >> 1 : dxy == 2 ? (s[0] + s[ss] + 1 - nr) >> 1
                                        : (s[0] + s[1] + s[ss] + s[ss + 1] + 2 - nr) >> 2);
        }
}

/* hpel_motion (:192-224): the 8x8 prediction of vector (mx, my) for the block at (x0, y0), into dst (stride 8) */
static void hpel_motion(const Ctx *c, uint8_t *dst, const uint8_t *ref, int x0, int y0, int mx, int my)
{
    uint8_t buf[9 * 16];
    int dxy = 0;
    const int sx = iclip(x0 + (mx >> 1), -16, c->width), sy = iclip(y0 + (my >> 1), -16, c->height);
    if (sx != c->width) dxy |= mx & 1;
    if (sy != c->height) dxy |= (my & 1) << 1;
    const uint8_t *s = ref + (ptrdiff_t)sy * c->ls + sx;
    ptrdiff_t ss = c->ls;
    if ((unsigned)sx > (unsigned)imax(c->h_edge - (mx & 1) - 8, 0) || (unsigned)sy > (unsigned)imax(c->v_edge - (my & 1) - 8, 0)) {
        s = emulate(buf, ref, c->ls, sx, sy, c->h_edge, c->v_edge);
        ss = 16;
    }
    put8(dst, 8, s, ss, dxy, c->no_rnd);
}

/* put_obmc's weights (:407-463) as rows of { top, left, mid, right, bottom } */
static void weights(int y, int x, int w[5])
{
    static const char *const rows[8] = {
        "22400 21500 21500 21500 20510 20510 20510 20420",
        "12500 12500 21500 21500 20510 20510 10520 10520",
        "12500 12500 11600 11600 10610 10610 10520 10520",
        "12500 12500 11600 11600 10610 10610 10520 10520",
        "02501 02501 01601 01601 00611 00611 00521 00521",
        "02501 02501 01601 01601 00611 00611 00521 00521",
        "02501 02501 01502 01502 00512 00512 00521 00521",
        "02402 01502 01502 01502 00512 00512 00512 00422",
    };
    for (int k = 0; k < 5; k++) w[k] = rows[y][6 * x + k] - '0';
}

/* chroma_4mv_motion (:577-627) with put / put_no_rnd */
static void chroma_4mv(const Ctx *c, uint8_t **dest, uint8_t **ref, int mb_x, int mb_y, int mx, int my)
{
    static const uint8_t tab[16] = { 0, 0, 0, 1, 1, 1, 1, 1, 0, 0, 0, 0, 0, 0, 1, 1 };
    uint8_t buf[9 * 16];
    mx = tab[mx & 15] + (mx >> 3);
    my = tab[my & 15] + (my >> 3);
    int dxy = ((my & 1) << 1) | (mx & 1);
    const int sx = iclip(mb_x * 8 + (mx >> 1), -8, c->width >> 1), sy = iclip(mb_y * 8 + (my >> 1), -8, c->height >> 1);
    if (sx == c->width >> 1) dxy &= ~1;
    if (sy == c->height >> 1) dxy &= ~2;
    const int emu = (unsigned)sx > (unsigned)imax((c->h_edge >> 1) - (dxy & 1) - 8, 0) ||
                    (unsigned)sy > (unsigned)imax((c->v_edge >> 1) - (dxy >> 1) - 8, 0);
    for (int p = 1; p < 3; p++) {
        const uint8_t *s = ref[p] + (ptrdiff_t)sy * c->uvls + sx;
        ptrdiff_t ss = c->uvls;
        if (emu) { s = emulate(buf, ref[p], c->uvls, sx, sy, c->h_edge >> 1, c->v_edge >> 1); ss = 16; }
        put8(dest[p], c->uvls, s, ss, dxy, c->no_rnd);
    }
}

int orc_mpvobmc_picture(uint8_t **dest, uint8_t **cur, uint8_t **last, uint8_t **next, const int *prm, const Rec *recs, size_t n,
                        const ObmcRec *obmc)
{
    if (prm[13]) return orc_mpvmc_picture(dest, cur, last, next, prm, recs, n);      /* B picture: obmc is ignored */
    const Ctx c = { prm[0], prm[1], prm[6], prm[7], prm[8], prm[9], prm[14] };
    const int mb_w = prm[4];
    for (size_t k = 0; k < n; k++) {
        const Rec *r = &recs[k];
        const ObmcRec *o = &obmc[k];
        if (!(r->mv_dir & 1)) continue;
        int16_t mc[4][4][2];                   /* mv_cache of :653-700 */
        const int top = r->mb_y > 0 && !(o->mb_type_top & 7), left = r->mb_x > 0 && !(o->mb_type_left & 7);
        const int right = r->mb_x + 1 < mb_w && !(o->mb_type_right & 7);
        for (int i = 0; i < 2; i++)
            for (int d = 0; d < 2; d++) {
                mc[1][1 + i][d] = o->mv[i][d];
                mc[2][1 + i][d] = mc[3][1 + i][d] = o->mv[2 + i][d];
                mc[0][1 + i][d] = top ? o->top[i][d] : mc[1][1 + i][d];
            }
        for (int i = 0; i < 2; i++)
            for (int d = 0; d < 2; d++) {
                mc[1 + i][0][d] = left ? o->left[i][d] : mc[1 + i][1][d];
                mc[1 + i][3][d] = right ? o->right[i][d] : mc[1 + i][2][d];
            }
        uint8_t *dy = dest[0] + (ptrdiff_t)r->mb_y * 16 * c.ls + r->mb_x * 16;
        int smx = 0, smy = 0;
        for (int b = 0; b < 4; b++) {
            const int x = (b & 1) + 1, y = (b >> 1) + 1, x0 = r->mb_x * 16 + (b & 1) * 8, y0 = r->mb_y * 16 + (b >> 1) * 8;
            const int16_t *v[5] = { mc[y][x], mc[y - 1][x], mc[y][x - 1], mc[y][x + 1], mc[y + 1][x] };   /* mid top left right bottom */
            uint8_t pred[5][64];
            for (int i = 0; i < 5; i++) hpel_motion(&c, pred[i], last[0], x0, y0, v[i][0], v[i][1]);
            uint8_t *d = dy + (b & 1) * 8 + (ptrdiff_t)(b >> 1) * 8 * c.ls;
            for (int yy = 0; yy < 8; yy++)
                for (int xx = 0; xx < 8; xx++) {
                    int w[5];
                    weights(yy, xx, w);
                    const int i = 8 * yy + xx;
                    d[yy * c.ls + xx] = (uint8_t)((w[0] * pred[1][i] + w[1] * pred[2][i] + w[2] * pred[0][i] + w[3] * pred[3][i] + w[4] * pred[4][i] + 4) >> 3);
                }
            smx += v[0][0];
            smy += v[0][1];
        }
        uint8_t *dc[3] = { dy, dest[1] + (ptrdiff_t)r->mb_y * 8 * c.uvls + r->mb_x * 8, dest[2] + (ptrdiff_t)r->mb_y * 8 * c.uvls + r->mb_x * 8 };
        chroma_4mv(&c, dc, last, r->mb_x, r->mb_y, smx, smy);
    }
    return 0;
}
