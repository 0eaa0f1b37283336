/*
 * oracle/refbuild/refapi_mpvmc.c -- TEST INFRASTRUCTURE, NOT PRODUCT.
 *
 * The reference's motion compensation for the mpegvideo decoders (libavcodec/mpegvideo_motion.c, compiled UNMODIFIED by Makefile into
 * oracle/_ref/libmpvmcref.so next to libavref.so).  libavref.so exports an aborting stand-in under the name ff_mpv_motion
 * (refapi_mpv_stubs.c); Makefile compiles the real function as ref_real_mpv_motion, so the two never meet.
 *
 * ref_mpvmc_picture() builds an MpegEncContext the way ff_mpv_frame_start() and mpeg_field_start() leave it for one picture (current /
 * last / next picture planes, doubled linesizes in a field picture, the DSP tables, an edge emulation buffer) and runs, per record, what
 * ff_mpv_reconstruct_mb() runs for an inter macroblock (mpegvideo.c:1548-1578): ff_mpv_motion for the forward direction with
 * put / put_no_rnd (h263dec.c:551-556 for the quarter-sample tables), then for the backward direction with avg.  A fresh context per
 * call, so calls on different pictures may run on different threads.  No arithmetic of its own.
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

/* prm: linesize, uvlinesize, pic_linesize, pic_uvlinesize, mb_width, mb_height, width, height, h_edge_pos, v_edge_pos, out_format
 * (0 FMT_MPEG1, 2 FMT_H263), picture_structure, first_field, b_picture, no_rounding, quarter_sample, workaround_bugs.
 * dest: current_picture.f->data (bottom field one line down); cur: current_picture_ptr->f->data; last / next: their pictures' data.
 * Every record is run: the caller passes only the records the product takes. */
int ref_mpvmc_picture(uint8_t **dest, uint8_t **cur, uint8_t **last, uint8_t **next, const int *prm, const Rec *recs, size_t n)
{
    enum { LS, UVLS, PLS, PUVLS, MBW, MBH, W, H, HE, VE, FMT, PS, FF, B, NR, QS, BUGS };
    AVCodecContext *avctx = calloc(1, sizeof(*avctx));
    MpegEncContext *s = calloc(1, sizeof(*s));
    AVFrame *fc = av_frame_alloc(), *fcp = av_frame_alloc(), *fl = av_frame_alloc(), *fn = av_frame_alloc();
    Picture *cur_ptr = calloc(1, sizeof(*cur_ptr));
    uint8_t *emu = malloc(64 * (size_t)prm[LS] + 64);
    if (!avctx || !s || !fc || !fcp || !fl || !fn || !cur_ptr || !emu) return -1;

    av_set_cpu_flags_mask(0);                     /* portable C only, like libavref.so */
    avctx->flags = AV_CODEC_FLAG_BITEXACT;
    s->avctx = avctx;
    ff_hpeldsp_init(&s->hdsp, avctx->flags);
    ff_qpeldsp_init(&s->qdsp);
    ff_videodsp_init(&s->vdsp, 8);
    s->out_format = prm[FMT] == 0 ? FMT_MPEG1 : FMT_H263;
    s->codec_id = prm[FMT] == 0 ? AV_CODEC_ID_MPEG2VIDEO : AV_CODEC_ID_MPEG4;
    s->chroma_x_shift = s->chroma_y_shift = 1;
    s->chroma_format = CHROMA_420;
    s->linesize = prm[LS]; s->uvlinesize = prm[UVLS];
    s->mb_width = prm[MBW]; s->mb_height = prm[MBH];
    s->width = prm[W]; s->height = prm[H];
    s->h_edge_pos = prm[HE]; s->v_edge_pos = prm[VE];
    s->picture_structure = prm[PS]; s->first_field = prm[FF];
    s->pict_type = prm[B] ? AV_PICTURE_TYPE_B : AV_PICTURE_TYPE_P;
    s->no_rounding = prm[NR]; s->quarter_sample = prm[QS]; s->workaround_bugs = prm[BUGS];
    s->sc.edge_emu_buffer = emu;

    for (int i = 0; i < 3; i++) {
        fc->data[i] = dest[i]; fcp->data[i] = cur[i]; fl->data[i] = last[i]; fn->data[i] = next[i];
        fc->linesize[i] = i ? prm[PUVLS] : prm[PLS];
        fcp->linesize[i] = fl->linesize[i] = fn->linesize[i] = fc->linesize[i];
    }
    s->current_picture.f = fc;
    cur_ptr->f = fcp;
    s->current_picture_ptr = cur_ptr;
    s->last_picture.f = fl;
    s->next_picture.f = fn;

    const int field_pic = s->picture_structure != PICT_FRAME;
    for (size_t i = 0; i < n; i++) {
        const Rec *r = &recs[i];
        s->mb_x = r->mb_x;
        s->mb_y = field_pic ? (r->mb_y << 1) | (s->picture_structure == PICT_BOTTOM_FIELD) : r->mb_y;
        s->mv_dir = r->mv_dir; s->mv_type = r->mv_type;
        for (int d = 0; d < 2; d++) {
            s->field_select[d][0] = r->field_select[d][0];
            s->field_select[d][1] = r->field_select[d][1];
            for (int k = 0; k < 4; k++) { s->mv[d][k][0] = r->mv[d][k][0]; s->mv[d][k][1] = r->mv[d][k][1]; }
        }
        /* s->dest[] as ff_init_block_index() sets it (mpegvideo.c:1730-1744) */
        const ptrdiff_t row = field_pic ? s->mb_y >> 1 : s->mb_y;
        uint8_t *dy = fc->data[0] + row * fc->linesize[0] * 16 + s->mb_x * 16;
        uint8_t *dcb = fc->data[1] + row * fc->linesize[1] * 8 + s->mb_x * 8;
        uint8_t *dcr = fc->data[2] + row * fc->linesize[2] * 8 + s->mb_x * 8;
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

    free(emu); free(cur_ptr);
    for (int i = 0; i < 3; i++) fc->data[i] = fcp->data[i] = fl->data[i] = fn->data[i] = NULL;
    av_frame_free(&fc); av_frame_free(&fcp); av_frame_free(&fl); av_frame_free(&fn);
    free(s); free(avctx);
    return 0;
}

/* the addresses of the function ref_mpvmc_picture runs and of the stand-in libavref.so exports as ff_mpv_motion: a test checks that they
 * differ (the stand-in aborts the process, so a picture that comes back at all was made by the real one) */
void ref_mpvmc_impl(void **real, void **stub)
{
    *real = (void *)ref_real_mpv_motion;
    *stub = (void *)ff_mpv_motion;
}
