/*
 * oracle/refbuild/refapi_xvid.c -- TEST INFRASTRUCTURE, NOT PRODUCT.
 *
 * The reference's Xvid IDCT (libavcodec/xvididct.c, compiled unmodified by Makefile into oracle/_ref/libxvidref.so next to
 * libavref.so) reached the way the MPEG-4 decoder reaches it: ff_xvid_idct_init() fills an IDCTDSPContext and every call goes
 * through that table.  ff_idctdsp_init() runs first, because xvid_idct_put / _add call the global ff_put_pixels_clamped /
 * ff_add_pixels_clamped, which only it sets.  No arithmetic of its own.
 */
#include <pthread.h>
#include <stdlib.h>
#include <string.h>

#include "libavutil/cpu.h"
#include "libavcodec/avcodec.h"
#include "libavcodec/idctdsp.h"
#include "libavcodec/xvididct.h"

static pthread_once_t once = PTHREAD_ONCE_INIT;
static IDCTDSPContext idsp, xvid;

static void init_all(void)
{
    AVCodecContext *avctx = calloc(1, sizeof(*avctx));
    av_set_cpu_flags_mask(0);                 /* portable C only, like libavref.so */
    avctx->bits_per_raw_sample = 8;
    avctx->idct_algo = FF_IDCT_AUTO;          /* what a decoder of an Xvid stream runs with */
    avctx->flags = AV_CODEC_FLAG_BITEXACT;
    ff_idctdsp_init(&idsp, avctx);
    xvid = idsp;                              /* what s->idsp holds when mpeg4videodec.c calls ff_xvid_idct_init */
    ff_xvid_idct_init(&xvid, avctx);
    free(avctx);
}
#define INIT() pthread_once(&once, init_all)

void ref_xvid_idct_put(uint8_t *d, ptrdiff_t s, int16_t *b) { INIT(); xvid.idct_put(d, s, b); }
void ref_xvid_idct_add(uint8_t *d, ptrdiff_t s, int16_t *b) { INIT(); xvid.idct_add(d, s, b); }
void ref_xvid_idct(int16_t *b) { INIT(); xvid.idct(b); }

/* mode 0 put, 1 add, 2 in place over n blocks, block i at frame + off[i] */
void ref_xvid_idct_batch(int mode, int16_t *blocks, uint8_t *frame, const uint32_t *off, ptrdiff_t stride, size_t n)
{
    INIT();
    for (size_t i = 0; i < n; i++) {
        int16_t *b = blocks + 64 * i;
        if (mode == 0)      xvid.idct_put(frame + off[i], stride, b);
        else if (mode == 1) xvid.idct_add(frame + off[i], stride, b);
        else                xvid.idct(b);
    }
}

/* Which entries does ff_xvid_idct_init fill in a zeroed IDCTDSPContext for (bits_per_raw_sample, idct_algo)?  out[i] = 1 when word i of
 * the six function pointers is non-zero; *perm_type and perm[64] are what it leaves there.  Returns the word count (6). */
int ref_xvid_table_fill(int bits, int algo, uint8_t *out, int *perm_type, uint8_t *perm)
{
    INIT();
    IDCTDSPContext c;
    AVCodecContext *avctx = calloc(1, sizeof(*avctx));
    memset(&c, 0, sizeof(c));
    avctx->bits_per_raw_sample = bits; avctx->idct_algo = algo; avctx->flags = AV_CODEC_FLAG_BITEXACT;
    ff_xvid_idct_init(&c, avctx);
    free(avctx);
    void *w[6];
    memcpy(w, &c, sizeof(w));
    for (int i = 0; i < 6; i++) out[i] = w[i] != NULL;
    *perm_type = (int)c.perm_type;
    memcpy(perm, c.idct_permutation, 64);
    return 6;
}
