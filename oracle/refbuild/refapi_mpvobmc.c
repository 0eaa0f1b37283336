/*
 * oracle/refbuild/refapi_mpvobmc.c -- TEST INFRASTRUCTURE, NOT PRODUCT.
 *
 * The reference's overlapped block motion compensation (apply_obmc in libavcodec/mpegvideo_motion.c, compiled UNMODIFIED by mpvobmc.mk
 * into oracle/_ref/libmpvobmcref.so next to libavref.so).  Like refapi_mpvmc.c, the real ff_mpv_motion is compiled under the name
 * ref_real_mpv_motion so that it never meets the aborting stand-in libavref.so exports.  No arithmetic of its own.
 */
#include <stdlib.h>
#include <string.h>

#include "libavutil/cpu.h"
#include "libavutil/frame.h"
#include "libavcodec/avcodec.h"
#include "libavcodec/mpegvideo.h"

void ref_real_mpv_motion(MpegEncContext *s, uint8_t *dest_y, uint8_t *dest_cb, uint8_t *dest_cr, int dir, uint8_t **ref_picture,
                         op_pixels_func (*pix_op)[4], qpel_mc_func (*qpix_op)[16]);

/* the 44-byte record of include/avdsp_b200.h (FFMpvMCRecord) */
typedef struct Rec {
    uint16_t mb_x, mb_y;
    uint8_t mv_dir, mv_type, field_select[2][2];
    int16_t mv[2][4][2];
    uint8_t pad[2];
} Rec;

/* the 52-byte record of include/avdsp_b200.h (FFMpvOBMCRecord): raw copies of what apply_obmc reads */
typedef struct ObmcRec {
    int16_t mv[4][2], top[2][2], left[2][2], right[2][2];
    uint32_t mb_type_top, mb_type_left, mb_type_right;
} ObmcRec;

/* ref_mpvmc_picture (refapi_mpvmc.c) with s->obmc = 1 (H.263 advanced prediction): current_picture.motion_val[0] / mb_type allocated with the strides and
 * offsets of the reference's picture tables (mpegpicture.c:249-253: b8_stride = 2 * mb_width + 1, motion_val = base + 4, mb_type = base
 * + 2 * mb_stride + 1) and an obmc_scratchpad.  Before each record, that record's raw entries are written where apply_obmc reads them
 * (mpegvideo_motion.c:653-700), so each macroblock sees what the decoder's tables held when it was reconstructed -- stale right
 * neighbours included -- and the real ff_mpv_motion runs.  In a B picture obmc is ignored, as there. */
int ref_mpvmc_obmc_picture(uint8_t **dest, uint8_t **cur, uint8_t **last, uint8_t **next, const int *prm, const Rec *recs, size_t n,
                           const ObmcRec *obmc)
{
    enum { LS, UVLS, PLS, PUVLS, MBW, MBH, W, H, HE, VE, FMT, PS, FF, B, NR, QS, BUGS };
    AVCodecContext *avctx = calloc(1, sizeof(*avctx));
    MpegEncContext *s = calloc(1, sizeof(*s));
    AVFrame *fc = av_frame_alloc(), *fcp = av_frame_alloc(), *fl = av_frame_alloc(), *fn = av_frame_alloc();
    Picture *cur_ptr = calloc(1, sizeof(*cur_ptr));
    uint8_t *emu = malloc(64 * (size_t)prm[LS] + 64), *scratch = malloc(32 * (size_t)prm[LS] + 64);
    const int mb_stride = prm[MBW] + 1, b8_stride = 2 * prm[MBW] + 1;
    int16_t (*mv_base)[2] = calloc((size_t)b8_stride * (2 * prm[MBH] + 4) + 8, sizeof(*mv_base));
    uint32_t *mbt_base = calloc((size_t)mb_stride * (prm[MBH] + 4) + 4, sizeof(*mbt_base));
    if (!avctx || !s || !fc || !fcp || !fl || !fn || !cur_ptr || !emu || !scratch || !mv_base || !mbt_base) return -1;

    av_set_cpu_flags_mask(0);
    avctx->flags = AV_CODEC_FLAG_BITEXACT;
    s->avctx = avctx;
    ff_hpeldsp_init(&s->hdsp, avctx->flags);
    ff_qpeldsp_init(&s->qdsp);
    ff_videodsp_init(&s->vdsp, 8);
    s->out_format = prm[FMT] == 0 ? FMT_MPEG1 : FMT_H263;
    s->codec_id = prm[FMT] == 0 ? AV_CODEC_ID_MPEG2VIDEO : AV_CODEC_ID_H263;
    s->chroma_x_shift = s->chroma_y_shift = 1;
    s->chroma_format = CHROMA_420;
    s->linesize = prm[LS]; s->uvlinesize = prm[UVLS];
    s->mb_width = prm[MBW]; s->mb_height = prm[MBH];
    s->mb_stride = mb_stride; s->b8_stride = b8_stride;
    s->width = prm[W]; s->height = prm[H];
    s->h_edge_pos = prm[HE]; s->v_edge_pos = prm[VE];
    s->picture_structure = prm[PS]; s->first_field = prm[FF];
    s->pict_type = prm[B] ? AV_PICTURE_TYPE_B : AV_PICTURE_TYPE_P;
    s->no_rounding = prm[NR]; s->quarter_sample = prm[QS]; s->workaround_bugs = prm[BUGS];
    s->obmc = 1;
    s->sc.edge_emu_buffer = emu;
    s->sc.obmc_scratchpad = scratch;

    for (int i = 0; i < 3; i++) {
        fc->data[i] = dest[i]; fcp->data[i] = cur[i]; fl->data[i] = last[i]; fn->data[i] = next[i];
        fc->linesize[i] = i ? prm[PUVLS] : prm[PLS];
        fcp->linesize[i] = fl->linesize[i] = fn->linesize[i] = fc->linesize[i];
    }
    s->current_picture.f = fc;
    s->current_picture.motion_val[0] = mv_base + 4;
    s->current_picture.mb_type = mbt_base + 2 * mb_stride + 1;
    cur_ptr->f = fcp;
    s->current_picture_ptr = cur_ptr;
    s->last_picture.f = fl;
    s->next_picture.f = fn;

    for (size_t i = 0; i < n; i++) {
        const Rec *r = &recs[i];
        const ObmcRec *o = &obmc[i];
        s->mb_x = r->mb_x;
        s->mb_y = r->mb_y;
        s->mv_dir = r->mv_dir; s->mv_type = r->mv_type;
        for (int d = 0; d < 2; d++) {
            s->field_select[d][0] = r->field_select[d][0];
            s->field_select[d][1] = r->field_select[d][1];
            for (int k = 0; k < 4; k++) { s->mv[d][k][0] = r->mv[d][k][0]; s->mv[d][k][1] = r->mv[d][k][1]; }
        }
        int16_t (*mv)[2] = s->current_picture.motion_val[0];
        const int mot_xy = 2 * s->mb_x + 2 * s->mb_y * b8_stride, xy = s->mb_x + s->mb_y * mb_stride;
        const int own[4] = { mot_xy, mot_xy + 1, mot_xy + b8_stride, mot_xy + b8_stride + 1 };
        for (int k = 0; k < 4; k++) { mv[own[k]][0] = o->mv[k][0]; mv[own[k]][1] = o->mv[k][1]; }
        if (s->mb_y) {
            for (int k = 0; k < 2; k++) { mv[mot_xy - b8_stride + k][0] = o->top[k][0]; mv[mot_xy - b8_stride + k][1] = o->top[k][1]; }
            s->current_picture.mb_type[xy - mb_stride] = o->mb_type_top;
        }
        if (s->mb_x) {
            for (int k = 0; k < 2; k++) { mv[mot_xy - 1 + k * b8_stride][0] = o->left[k][0]; mv[mot_xy - 1 + k * b8_stride][1] = o->left[k][1]; }
            s->current_picture.mb_type[xy - 1] = o->mb_type_left;
        }
        if (s->mb_x + 1 < s->mb_width) {
            for (int k = 0; k < 2; k++) { mv[mot_xy + 2 + k * b8_stride][0] = o->right[k][0]; mv[mot_xy + 2 + k * b8_stride][1] = o->right[k][1]; }
            s->current_picture.mb_type[xy + 1] = o->mb_type_right;
        }
        uint8_t *dy = fc->data[0] + (ptrdiff_t)s->mb_y * fc->linesize[0] * 16 + s->mb_x * 16;
        uint8_t *dcb = fc->data[1] + (ptrdiff_t)s->mb_y * fc->linesize[1] * 8 + s->mb_x * 8;
        uint8_t *dcr = fc->data[2] + (ptrdiff_t)s->mb_y * fc->linesize[2] * 8 + s->mb_x * 8;
        op_pixels_func (*op_pix)[4];
        qpel_mc_func (*op_qpix)[16];
        if (!s->no_rounding || s->pict_type == AV_PICTURE_TYPE_B) {
            op_pix = s->hdsp.put_pixels_tab; op_qpix = s->qdsp.put_qpel_pixels_tab;
        } else {
            op_pix = s->hdsp.put_no_rnd_pixels_tab; op_qpix = s->qdsp.put_no_rnd_qpel_pixels_tab;
        }
        if (s->mv_dir & MV_DIR_FORWARD) {
            ref_real_mpv_motion(s, dy, dcb, dcr, 0, s->last_picture.f->data, op_pix, op_qpix);
            op_pix = s->hdsp.avg_pixels_tab;
            op_qpix = s->qdsp.avg_qpel_pixels_tab;
        }
        if (s->mv_dir & MV_DIR_BACKWARD)
            ref_real_mpv_motion(s, dy, dcb, dcr, 1, s->next_picture.f->data, op_pix, op_qpix);
    }

    free(emu); free(scratch); free(cur_ptr); free(mv_base); free(mbt_base);
    for (int i = 0; i < 3; i++) fc->data[i] = fcp->data[i] = fl->data[i] = fn->data[i] = NULL;
    av_frame_free(&fc); av_frame_free(&fcp); av_frame_free(&fl); av_frame_free(&fn);
    free(s); free(avctx);
    return 0;
}
