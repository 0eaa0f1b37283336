/*
 * oracle/port/orc_h263.c -- TEST INFRASTRUCTURE, NOT PRODUCT.
 *
 * CPU restatement (plain C) of the H.263 deblocking filter: the two H263DSPContext edge filters (libavcodec/h263dsp.c:31-115) and the
 * picture filter ff_h263_loop_filter (h263.c:135-220) run for every macroblock in raster order -- restated here not in that serial order
 * but as the two passes the product runs: every horizontal edge (h263_v_loop_filter) of the picture, then every vertical edge
 * (h263_h_loop_filter), with each edge's qp a function of its two macroblocks alone:
 *   qp_c(M) = IS_SKIP(mb_type[M]) ? 0 : qscale_table[M], 0 meaning "not filtered";
 *   luma edges inside M (row 16Y+8, column 16X+8): qp_c(M);
 *   the top edge of M (Y > 0) and its left edge (X > 0), luma and chroma: qp_c(M) ? qp_c(M) : qp_c(above / left);
 *   chroma edges filter with chroma_qscale_table[qp]; the picture's bottom and right borders are never filtered.
 * tests/test_h263_cpu.py pins this against the serial reference driver (oracle/refbuild/refapi_h263.c), which is the proof that the
 * serial order and the two passes give the same bytes.  Same arguments as ref_h263_loop_filter_picture.
 */
#include <stdint.h>
#include <stddef.h>

static const uint8_t strength_tab[32] = {
    0, 1, 1, 2, 2, 3, 3, 4, 4, 4, 5, 5, 6, 6, 7, 7, 7, 8, 8, 8, 9, 9, 9, 10, 10, 10, 11, 11, 11, 12, 12, 12
};

/* one line across the edge between p[-step] and p[0] */
static void filter_line(uint8_t *p, ptrdiff_t step, int strength)
{
    const int p0 = p[-2 * step], p1 = p[-step], p2 = p[0], p3 = p[step];
    const int d = (p0 - p3 + 4 * (p2 - p1)) / 8;
    int d1, q1, q2, ad1, d2;
    if (d < -2 * strength)   d1 = 0;
    else if (d < -strength)  d1 = -2 * strength - d;
    else if (d < strength)   d1 = d;
    else if (d < 2 * strength) d1 = 2 * strength - d;
    else                     d1 = 0;
    q1 = p1 + d1;
    q2 = p2 - d1;
    if (q1 & 256) q1 = ~(q1 >> 31);
    if (q2 & 256) q2 = ~(q2 >> 31);
    ad1 = (d1 < 0 ? -d1 : d1) >> 1;
    d2 = (p0 - p3) / 4;
    if (d2 < -ad1) d2 = -ad1;
    if (d2 > ad1) d2 = ad1;
    p[-2 * step] = (uint8_t)(p0 - d2);
    p[-step] = (uint8_t)q1;
    p[0] = (uint8_t)q2;
    p[step] = (uint8_t)(p3 + d2);
}

/* H263DSPContext.h263_h_loop_filter: the vertical edge left of src, 8 rows */
void orc_h263_h_loop_filter(uint8_t *src, int stride, int qscale)
{
    for (int y = 0; y < 8; y++) filter_line(src + y * stride, 1, strength_tab[qscale]);
}

/* H263DSPContext.h263_v_loop_filter: the horizontal edge above src, 8 columns */
void orc_h263_v_loop_filter(uint8_t *src, int stride, int qscale)
{
    for (int x = 0; x < 8; x++) filter_line(src + x, stride, strength_tab[qscale]);
}

typedef struct Pic {
    const uint32_t *mb_type;
    const int8_t *qscale;
    int mb_stride;
} Pic;

static int qp_c(const Pic *p, int x, int y)
{
    const int i = x + y * p->mb_stride;
    return (p->mb_type[i] & (1 << 11)) ? 0 : p->qscale[i];
}

/* the qp of the edge in front of 8-sample block a of a plane (a >= 1) whose macroblocks are 8 << luma samples wide; (mx, my) is the
 * macroblock after the edge and (px, py) the one before it */
static int edge_qp(const Pic *p, int luma, int a, int mx, int my, int px, int py)
{
    const int q = qp_c(p, mx, my);
    if (luma && (a & 1)) return q;              /* inside a luma macroblock */
    return q ? q : qp_c(p, px, py);
}

/* prm: linesize, uvlinesize, mb_width, mb_height, mb_stride */
int orc_h263_loop_filter_picture(uint8_t **data, const int *prm, const uint32_t *mb_type, const int8_t *qscale_table,
                                 const uint8_t *chroma_qscale_table)
{
    const Pic P = { mb_type, qscale_table, prm[4] };
    for (int pl = 0; pl < 3; pl++) {
        const int luma = pl == 0, ls = luma ? prm[0] : prm[1];
        const int nbx = prm[2] << luma, nby = prm[3] << luma;     /* 8-sample blocks across / down */
        uint8_t *base = data[pl];
        /* pass 1: horizontal edges */
        for (int a = 1; a < nby; a++)
            for (int b = 0; b < nbx; b++) {
                const int mx = b >> luma, my = a >> luma;
                int q = edge_qp(&P, luma, a, mx, my, mx, my - 1);
                if (!q) continue;
                if (!luma) q = chroma_qscale_table[q];
                orc_h263_v_loop_filter(base + (ptrdiff_t)8 * a * ls + 8 * b, ls, q);
            }
        /* pass 2: vertical edges */
        for (int b = 0; b < nby; b++)
            for (int a = 1; a < nbx; a++) {
                const int mx = a >> luma, my = b >> luma;
                int q = edge_qp(&P, luma, a, mx, my, mx - 1, my);
                if (!q) continue;
                if (!luma) q = chroma_qscale_table[q];
                orc_h263_h_loop_filter(base + (ptrdiff_t)8 * b * ls + 8 * a, ls, q);
            }
    }
    return 0;
}
