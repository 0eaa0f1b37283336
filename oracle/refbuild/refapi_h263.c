/*
 * oracle/refbuild/refapi_h263.c -- TEST INFRASTRUCTURE, NOT PRODUCT.
 *
 * The reference's H.263 deblocking filter (libavcodec/h263dsp.c and the per-macroblock driver ff_h263_loop_filter of
 * libavcodec/h263.c, both compiled UNMODIFIED by h263.mk into oracle/_ref/libh263ref.so next to libavref.so).  No arithmetic of its own.
 *
 * ref_h263_loop_filter_picture() runs ff_h263_loop_filter for every macroblock of one picture in raster order, as h263dec.c decode_slice
 * (:250-252, :281-283) and rv10.c (:654-655) do after each ff_mpv_reconstruct_mb: s->dest as ff_init_block_index / ff_update_block_index
 * set it, and s->qscale = qscale_table[xy], the value ff_mpv_reconstruct_mb has just stored there (mpegvideo.c:1490).  A fresh context
 * per call, so calls on different pictures may run on different threads.
 */
#include <stddef.h>
#include <stdlib.h>
#include <string.h>

#include "libavutil/frame.h"
#include "libavcodec/avcodec.h"
#include "libavcodec/h263.h"
#include "libavcodec/h263dsp.h"
#include "libavcodec/mpegvideo.h"

/* prm: linesize, uvlinesize, mb_width, mb_height, mb_stride */
int ref_h263_loop_filter_picture(uint8_t **data, const int *prm, uint32_t *mb_type, int8_t *qscale_table, const uint8_t *chroma_qscale_table)
{
    AVCodecContext *avctx = calloc(1, sizeof(*avctx));
    MpegEncContext *s = calloc(1, sizeof(*s));
    AVFrame *f = av_frame_alloc();
    if (!avctx || !s || !f) return -1;
    s->avctx = avctx;
    s->linesize = prm[0]; s->uvlinesize = prm[1];
    s->mb_width = prm[2]; s->mb_height = prm[3]; s->mb_stride = prm[4];
    s->b8_stride = 2 * s->mb_width + 1;
    s->chroma_x_shift = s->chroma_y_shift = 1;
    s->picture_structure = PICT_FRAME;
    s->pict_type = AV_PICTURE_TYPE_P;
    s->chroma_qscale_table = chroma_qscale_table;
    ff_h263dsp_init(&s->h263dsp);
    for (int i = 0; i < 3; i++) {
        f->data[i] = data[i];
        f->linesize[i] = i ? prm[1] : prm[0];
    }
    s->current_picture.f = f;
    s->current_picture.mb_type = mb_type;
    s->current_picture.qscale_table = qscale_table;

    for (s->mb_y = 0; s->mb_y < s->mb_height; s->mb_y++) {
        s->mb_x = 0;                                  /* ff_init_block_index reads it (h263dec.c:283-289 resets it per row) */
        ff_init_block_index(s);
        for (; s->mb_x < s->mb_width; s->mb_x++) {
            ff_update_block_index(s);
            s->qscale = qscale_table[s->mb_x + s->mb_y * s->mb_stride];
            ff_h263_loop_filter(s);
        }
    }

    for (int i = 0; i < 3; i++) f->data[i] = NULL;
    av_frame_free(&f);
    free(s); free(avctx);
    return 0;
}

/* the table ff_h263dsp_init fills */
void ref_h263dsp_init(H263DSPContext *c)
{
    ff_h263dsp_init(c);
}

/* sizeof(H263DSPContext) and the offsets of its two slots */
void ref_h263_abi_info(int *out)
{
    out[0] = (int)sizeof(H263DSPContext);
    out[1] = (int)offsetof(H263DSPContext, h263_h_loop_filter);
    out[2] = (int)offsetof(H263DSPContext, h263_v_loop_filter);
}
