/*
 * oracle/refbuild/refapi_mpvgmc.c -- TEST INFRASTRUCTURE, NOT PRODUCT.
 *
 * The reference's motion compensation on MPEG-4 S-VOPs: libavcodec/mpegvideo_motion.c compiled UNMODIFIED (as ref_real_mpv_motion, the
 * object libmpvmcref.so links) into oracle/_ref/libmpvgmcref.so by mpvgmc.mk.  ref_mpvmc_gmc_picture() builds an MpegEncContext the way
 * ff_mpv_frame_start() leaves it for one S-VOP -- the frame planes, the DSP tables with MpegVideoDSPContext from ff_mpegvideodsp_init
 * (mpegvideo.c:274), pict_type AV_PICTURE_TYPE_S and the sprite fields mpeg4_decode_sprite_trajectory sets -- and runs, per record, what
 * ff_mpv_reconstruct_mb() runs for an inter macroblock (mpegvideo.c:1548-1578) with s->mcsel taken from the record: ff_mpv_motion for the
 * forward direction with put / put_no_rnd, then for the backward direction with avg.  The context set-up is that of refapi_mpvmc.c for a
 * frame picture.  A fresh context per call, so calls on different pictures may run on different threads.  No arithmetic of its own.
 */
#include <stddef.h>
#include <stdlib.h>
#include <string.h>

#include "libavutil/cpu.h"
#include "libavutil/frame.h"
#include "libavcodec/avcodec.h"
#include "libavcodec/mpegvideo.h"
#include "libavcodec/mpegvideodsp.h"

void ref_real_mpv_motion(MpegEncContext *s, uint8_t *dest_y, uint8_t *dest_cb, uint8_t *dest_cr, int dir, uint8_t **ref_picture,
                         op_pixels_func (*pix_op)[4], qpel_mc_func (*qpix_op)[16]);

/* the 44-byte record of include/avdsp_b200.h (FFMpvMCRecord) */
typedef struct Rec {
    uint16_t mb_x, mb_y;
    uint8_t mv_dir, mv_type, field_select[2][2];
    int16_t mv[2][4][2];
    uint8_t mcsel, pad;
} Rec;

/* prm: as ref_mpvmc_picture's (refapi_mpvmc.c); the picture must be a frame picture.  sprite: sprite_warping_accuracy,
 * real_sprite_warping_points, sprite_offset[2][2], sprite_delta[2][2].  Every record is run: the caller passes only the records the
 * product takes. */
int ref_mpvmc_gmc_picture(uint8_t **dest, uint8_t **cur, uint8_t **last, uint8_t **next, const int *prm, const Rec *recs, size_t n,
                          const int *sprite)
{
    enum { LS, UVLS, PLS, PUVLS, MBW, MBH, W, H, HE, VE, FMT, PS, FF, B, NR, QS, BUGS };
    if (prm[PS] != PICT_FRAME) return -1;
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
    ff_mpegvideodsp_init(&s->mdsp);
    s->out_format = FMT_H263;
    s->codec_id = AV_CODEC_ID_MPEG4;
    s->chroma_x_shift = s->chroma_y_shift = 1;
    s->chroma_format = CHROMA_420;
    s->linesize = prm[LS]; s->uvlinesize = prm[UVLS];
    s->mb_width = prm[MBW]; s->mb_height = prm[MBH];
    s->width = prm[W]; s->height = prm[H];
    s->h_edge_pos = prm[HE]; s->v_edge_pos = prm[VE];
    s->picture_structure = PICT_FRAME; s->first_field = prm[FF];
    s->pict_type = AV_PICTURE_TYPE_S;
    s->no_rounding = prm[NR]; s->quarter_sample = prm[QS]; s->workaround_bugs = prm[BUGS];
    s->sc.edge_emu_buffer = emu;
    s->sprite_warping_accuracy = sprite[0];
    s->real_sprite_warping_points = sprite[1];
    for (int i = 0; i < 2; i++)
        for (int k = 0; k < 2; k++) { s->sprite_offset[i][k] = sprite[2 + 2 * i + k]; s->sprite_delta[i][k] = sprite[6 + 2 * i + k]; }

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

    for (size_t i = 0; i < n; i++) {
        const Rec *r = &recs[i];
        s->mb_x = r->mb_x;
        s->mb_y = r->mb_y;
        s->mv_dir = r->mv_dir; s->mv_type = r->mv_type;
        s->mcsel = r->mcsel;
        for (int d = 0; d < 2; d++) {
            s->field_select[d][0] = r->field_select[d][0];
            s->field_select[d][1] = r->field_select[d][1];
            for (int k = 0; k < 4; k++) { s->mv[d][k][0] = r->mv[d][k][0]; s->mv[d][k][1] = r->mv[d][k][1]; }
        }
        /* s->dest[] as ff_init_block_index() sets it (mpegvideo.c:1730-1744) */
        uint8_t *dy = fc->data[0] + (ptrdiff_t)s->mb_y * fc->linesize[0] * 16 + s->mb_x * 16;
        uint8_t *dcb = fc->data[1] + (ptrdiff_t)s->mb_y * fc->linesize[1] * 8 + s->mb_x * 8;
        uint8_t *dcr = fc->data[2] + (ptrdiff_t)s->mb_y * fc->linesize[2] * 8 + s->mb_x * 8;
        op_pixels_func (*op_pix)[4];
        qpel_mc_func (*op_qpix)[16];
        if (!s->no_rounding) {
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

/* the table ff_mpegvideodsp_init fills, and sizeof(MpegVideoDSPContext) with the offsets of its two slots */
void ref_mpegvideodsp_init(MpegVideoDSPContext *c)
{
    ff_mpegvideodsp_init(c);
}

void ref_mpegvideodsp_layout(int *out)
{
    out[0] = (int)sizeof(MpegVideoDSPContext);
    out[1] = (int)offsetof(MpegVideoDSPContext, gmc1);
    out[2] = (int)offsetof(MpegVideoDSPContext, gmc);
}
