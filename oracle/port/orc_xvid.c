/*
 * oracle/port/orc_xvid.c -- TEST INFRASTRUCTURE, NOT PRODUCT.
 *
 * CPU restatement (plain C) of the reference's Xvid 8x8 IDCT, ff_xvid_idct / xvid_idct_put / xvid_idct_add
 * (libavcodec/xvididct.c:40-331), in its formula-wise form: every row through the general 4 + 4-term formula of idct_row
 * (:118-138) with the one exception its `return 0` makes (row 0 = {-4, 0, ...} is left as it was), every column through
 * idct_col_8 (:162-206).  Pinned block for block against oracle/_ref/libxvidref.so (the unmodified xvididct.c) and against
 * the known answers of the reference's own IDCT test (tests/golden/fate_idct8x8_xvid.txt) by tests/test_xvid_idct.py.
 * Arithmetic is uint32_t where the reference uses int, so that the 32-bit overflow of full-range input wraps as it does
 * there instead of being undefined.
 */
#include <stdint.h>
#include <stddef.h>
#include <pthread.h>

static const uint32_t TAB[4][7] = {
    { 22725, 21407, 19266, 16384, 12873,  8867, 4520 },    /* TAB04 */
    { 31521, 29692, 26722, 22725, 17855, 12299, 6270 },    /* TAB17 */
    { 29692, 27969, 25172, 21407, 16819, 11585, 5906 },    /* TAB26 */
    { 26722, 25172, 22654, 19266, 15137, 10426, 5315 },    /* TAB35 */
};
static const int ROW_TAB[8] = { 0, 1, 2, 3, 0, 3, 2, 1 };
static const uint32_t RND[8] = { 65536, 3597, 2260, 1203, 0, 120, 512, 512 };

static inline int sra(uint32_t v, int s) { return (int32_t)v >> s; }
static inline uint8_t clamp_u8(int v) { return v < 0 ? 0 : v > 255 ? 255 : (uint8_t)v; }

static void xvid_row(int16_t *in, int r)
{
    const uint32_t *c = TAB[ROW_TAB[r]];
    if (r == 0 && in[0] == -4 && !(in[1] | in[2] | in[3] | in[4] | in[5] | in[6] | in[7]))
        return;                                                 /* (16384 * -4 + 65536) >> 11 == 0: idct_row returns 0 */
    const uint32_t x0 = in[0], x1 = in[1], x2 = in[2], x3 = in[3], x4 = in[4], x5 = in[5], x6 = in[6], x7 = in[7];
    const uint32_t k = c[3] * x0 + RND[r];
    const uint32_t a0 = k + c[1] * x2 + c[3] * x4 + c[5] * x6;
    const uint32_t a1 = k + c[5] * x2 - c[3] * x4 - c[1] * x6;
    const uint32_t a2 = k - c[5] * x2 - c[3] * x4 + c[1] * x6;
    const uint32_t a3 = k - c[1] * x2 + c[3] * x4 - c[5] * x6;
    const uint32_t b0 = c[0] * x1 + c[2] * x3 + c[4] * x5 + c[6] * x7;
    const uint32_t b1 = c[2] * x1 - c[6] * x3 - c[0] * x5 - c[4] * x7;
    const uint32_t b2 = c[4] * x1 - c[0] * x3 + c[6] * x5 + c[2] * x7;
    const uint32_t b3 = c[6] * x1 - c[4] * x3 + c[2] * x5 - c[0] * x7;
    in[0] = (int16_t)sra(a0 + b0, 11); in[7] = (int16_t)sra(a0 - b0, 11);
    in[1] = (int16_t)sra(a1 + b1, 11); in[6] = (int16_t)sra(a1 - b1, 11);
    in[2] = (int16_t)sra(a2 + b2, 11); in[5] = (int16_t)sra(a2 - b2, 11);
    in[3] = (int16_t)sra(a3 + b3, 11); in[4] = (int16_t)sra(a3 - b3, 11);
}

static inline uint32_t mult(uint32_t c, uint32_t x) { return (uint32_t)sra(c * x, 16); }

static void xvid_col(int16_t *in)
{
    enum { TAN1 = 0x32EC, TAN2 = 0x6A0A, TAN3 = 0xAB0E, SQRT2 = 0x5A82 };
    const uint32_t x0 = in[0], x1 = in[8], x2 = in[16], x3 = in[24], x4 = in[32], x5 = in[40], x6 = in[48], x7 = in[56];
    const uint32_t m0 = mult(TAN1, x7) + x1, m1 = mult(TAN1, x1) - x7, m2 = mult(TAN3, x5) + x3, m3 = mult(TAN3, x3) - x5;
    const uint32_t t7 = m0 + m2, t4 = m1 - m3, t0 = m0 - m2, t1 = m1 + m3;
    const uint32_t t6 = 2 * mult(SQRT2, t0 + t1), t5 = 2 * mult(SQRT2, t0 - t1);
    const uint32_t e3 = mult(TAN2, x6) + x2, e2 = mult(TAN2, x2) - x6, e0 = x0 + x4, e1 = x0 - x4;
    const uint32_t a0 = e0 + e3, a3 = e0 - e3, a1 = e1 + e2, a2 = e1 - e2;
    in[0]  = (int16_t)sra(a0 + t7, 6); in[56] = (int16_t)sra(a0 - t7, 6);
    in[24] = (int16_t)sra(a3 + t4, 6); in[32] = (int16_t)sra(a3 - t4, 6);
    in[8]  = (int16_t)sra(a1 + t6, 6); in[48] = (int16_t)sra(a1 - t6, 6);
    in[16] = (int16_t)sra(a2 + t5, 6); in[40] = (int16_t)sra(a2 - t5, 6);
}

void orc_xvid_idct(int16_t *block)
{
    for (int r = 0; r < 8; r++) xvid_row(block + 8 * r, r);
    for (int c = 0; c < 8; c++) xvid_col(block + c);
}

/* ff_xvid_idct followed by put / add_pixels_clamped (idctdsp.c:85-145), as xvid_idct_put / _add do (:321-331) */
void orc_xvid_idct_put(uint8_t *dst, ptrdiff_t stride, int16_t *block)
{
    orc_xvid_idct(block);
    for (int y = 0; y < 8; y++)
        for (int x = 0; x < 8; x++) dst[y * stride + x] = clamp_u8(block[8 * y + x]);
}

void orc_xvid_idct_add(uint8_t *dst, ptrdiff_t stride, int16_t *block)
{
    orc_xvid_idct(block);
    for (int y = 0; y < 8; y++)
        for (int x = 0; x < 8; x++) dst[y * stride + x] = clamp_u8(dst[y * stride + x] + block[8 * y + x]);
}

/* ---- batch driver, the shape of orc_idct_batch: mode 0 put, 1 add, 2 in place; the block range split over pthreads ---- */
struct xvid_span { int mode; int16_t *blocks; uint8_t *frame; const uint32_t *off; ptrdiff_t stride; size_t lo, hi; };
static void *xvid_span_run(void *arg)
{
    struct xvid_span *s = arg;
    for (size_t i = s->lo; i < s->hi; i++) {
        int16_t *b = s->blocks + 64 * i;
        if (s->mode == 0)      orc_xvid_idct_put(s->frame + s->off[i], s->stride, b);
        else if (s->mode == 1) orc_xvid_idct_add(s->frame + s->off[i], s->stride, b);
        else                   orc_xvid_idct(b);
    }
    return NULL;
}
void orc_xvid_idct_batch(int mode, int16_t *blocks, uint8_t *frame, const uint32_t *dst_off, ptrdiff_t stride, size_t n, int nthreads)
{
    enum { MAXT = 256 };
    pthread_t th[MAXT];
    struct xvid_span sp[MAXT];
    if (nthreads < 1) nthreads = 1;
    if (nthreads > MAXT) nthreads = MAXT;
    for (int t = 0; t < nthreads; t++) {
        sp[t] = (struct xvid_span){ mode, blocks, frame, dst_off, stride, n * t / nthreads, n * (t + 1) / nthreads };
        if (nthreads > 1) pthread_create(&th[t], NULL, xvid_span_run, &sp[t]);
        else xvid_span_run(&sp[t]);
    }
    if (nthreads > 1) for (int t = 0; t < nthreads; t++) pthread_join(th[t], NULL);
}
