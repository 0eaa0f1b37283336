/*
 * examples/reference_binding/dsp_init_cuda.c -- the file a libav maintainer would add as libavcodec/cuda/dsp_init_cuda.c +
 * libswscale/cuda/swscale_cuda.c (INTEGRATION.md sections 2 and 4), written against the REFERENCE'S OWN headers: it is compiled in the
 * CPU test-suite with -I/root/reference (tests/test_abi_cpu.py::test_reference_side_binding_compiles) so that every hook prototype and
 * every slot assignment is type-checked against the reference's real struct definitions, not against this repository's mirrors.
 * Nothing here computes anything: each function forwards to libavdsp_b200.so.
 */
#include <stdint.h>
#include <stddef.h>

#include "libavcodec/avcodec.h"
#include "libavcodec/idctdsp.h"
#include "libavcodec/fdctdsp.h"
#include "libavcodec/faandct.h"
#include "libavcodec/blockdsp.h"
#include "libavcodec/me_cmp.h"
#include "libavcodec/mpegvideodsp.h"
#include "libavcodec/h263dsp.h"
#include "libavcodec/h264dsp.h"
#include "libavcodec/h264qpel.h"
#include "libavcodec/h264chroma.h"
#include "libavcodec/h264pred.h"
#include "libavcodec/hpeldsp.h"
#include "libavcodec/pixblockdsp.h"
#include "libavcodec/proresdsp.h"
#include "libavcodec/qpeldsp.h"
#include "libavcodec/fft.h"
#include "libswscale/swscale.h"
#include "libswscale/swscale_internal.h"

/* ---- prototypes of include/avdsp_b200.h, repeated so that the reference's struct definitions are the ones in scope ---- */
int  avb200_init(int device);
void ff_idctdsp_init_cuda(IDCTDSPContext *c, int idct_algo, int bits_per_raw_sample, unsigned high_bit_depth);
void ff_xvid_idct_init_cuda(IDCTDSPContext *c, int idct_algo, int bits_per_raw_sample);
void ff_fdctdsp_init_cuda(FDCTDSPContext *c, int dct_algo, int bits_per_raw_sample, unsigned high_bit_depth);
void ff_blockdsp_init_cuda(BlockDSPContext *c);
void ff_me_cmp_init_cuda(MECmpContext *c);
void ff_h264dsp_init_cuda(H264DSPContext *c, const int bit_depth, const int chroma_format_idc);
void ff_h264qpel_init_cuda(H264QpelContext *c, int bit_depth);
void ff_h264chroma_init_cuda(H264ChromaContext *c, int bit_depth);
void ff_h264_pred_init_cuda(H264PredContext *h, int codec_id, const int bit_depth, const int chroma_format_idc);
void ff_hpeldsp_init_cuda(HpelDSPContext *c, int flags);
void ff_pixblockdsp_init_cuda(PixblockDSPContext *c, unsigned high_bit_depth);
void ff_qpeldsp_init_cuda(QpelDSPContext *c);
void ff_h263dsp_init_cuda(H263DSPContext *c);
void ff_mpegvideodsp_init_cuda(MpegVideoDSPContext *c);
void ff_proresdsp_init_cuda(ProresDSPContext *dsp);
void ff_fft_init_cuda(FFTContext *s);
void ff_mdct_init_cuda(FFTContext *s);

typedef struct SwsContextCUDA SwsContextCUDA;
SwsContextCUDA *sws_getContext_cuda(int srcW, int srcH, int srcFormat, int dstW, int dstH, int dstFormat, int flags,
                                    void *srcFilter, void *dstFilter, const double *param);
void sws_freeContext_cuda(SwsContextCUDA *ctx);
int  sws_setColorspaceDetails_cuda(SwsContextCUDA *ctx, const int inv_table[4], int srcRange, const int table[4], int dstRange,
                                   int brightness, int contrast, int saturation);
int  sws_scale_cuda(SwsContextCUDA *ctx, const uint8_t *const srcSlice[], const int srcStride[], int srcSliceY, int srcSliceH,
                    uint8_t *const dst[], const int dstStride[]);
/* the slot table of include/avdsp_b200.h, here with the reference's own function-pointer typedefs (swscale_internal.h:62-110): the
 * assignments below only compile if the two declarations agree */
typedef struct SwsLineSlotsCUDA {
    void (*hyScale)(struct SwsContext *c, int16_t *dst, int dstW, const uint8_t *src, const int16_t *filter, const int32_t *filterPos, int filterSize);
    void (*hcScale)(struct SwsContext *c, int16_t *dst, int dstW, const uint8_t *src, const int16_t *filter, const int32_t *filterPos, int filterSize);
    void (*hyscale_fast)(struct SwsContext *c, int16_t *dst, int dstWidth, const uint8_t *src, int srcW, int xInc);
    void (*hcscale_fast)(struct SwsContext *c, int16_t *dst1, int16_t *dst2, int dstWidth, const uint8_t *src1, const uint8_t *src2, int srcW, int xInc);
    yuv2planar1_fn yuv2plane1;
    yuv2planarX_fn yuv2planeX;
    yuv2interleavedX_fn yuv2nv12cX;
    yuv2packed1_fn yuv2packed1;
    yuv2packed2_fn yuv2packed2;
    yuv2packedX_fn yuv2packedX;
    void (*lumConvertRange)(int16_t *dst, int width);
    void (*chrConvertRange)(int16_t *dst1, int16_t *dst2, int width);
} SwsLineSlotsCUDA;
int ff_sws_init_swscale_cuda(struct SwsContext *c, SwsContextCUDA *cuda, SwsLineSlotsCUDA *slots);

/* ---- libavcodec: one call next to each existing arch hook (INTEGRATION.md section 2) ---- */
void ff_idctdsp_init_cuda_hook(IDCTDSPContext *c, AVCodecContext *avctx, unsigned high_bit_depth)      /* idctdsp.c:183-188 */
{
    ff_idctdsp_init_cuda(c, avctx->idct_algo, avctx->bits_per_raw_sample, high_bit_depth);
}
/* mpeg4videodec.c:2084-2085 and :2558-2559, right after each ff_xvid_idct_init(&s->idsp, avctx) */
void ff_xvid_idct_init_cuda_hook(IDCTDSPContext *c, AVCodecContext *avctx)
{
    ff_xvid_idct_init_cuda(c, avctx->idct_algo, avctx->bits_per_raw_sample);
}
void ff_fdctdsp_init_cuda_hook(FDCTDSPContext *c, AVCodecContext *avctx, unsigned high_bit_depth)      /* fdctdsp.c:45-48 */
{
    ff_fdctdsp_init_cuda(c, avctx->dct_algo, avctx->bits_per_raw_sample, high_bit_depth);
}
void ff_pixblockdsp_init_cuda_hook(PixblockDSPContext *c, AVCodecContext *avctx, unsigned high_bit_depth)      /* pixblockdsp.c:70-77 */
{
    (void)avctx;
    ff_pixblockdsp_init_cuda(c, high_bit_depth);
}
/* proresdsp.c:76-77: in place of ff_proresdsp_init_x86(dsp), before ff_init_scantable_permutation(); the CUDA slot wants
 * FF_IDCT_PERM_NONE, the order of the C function, not the x86 code's transposed one */
void ff_proresdsp_init_cuda_hook(ProresDSPContext *dsp)
{
    ff_proresdsp_init_cuda(dsp);
}
/* the remaining tables take exactly the arguments of their x86 hooks: ff_blockdsp_init_cuda(c), ff_me_cmp_init_cuda(c),
 * ff_h264dsp_init_cuda(c, bit_depth, chroma_format_idc), ff_h264qpel_init_cuda(c, bit_depth), ff_h264chroma_init_cuda(c, bit_depth),
 * ff_h264_pred_init_cuda(h, codec_id, bit_depth, chroma_format_idc), ff_hpeldsp_init_cuda(c, flags), ff_qpeldsp_init_cuda(c),
 * ff_fft_init_cuda(s), ff_mdct_init_cuda(s), ff_h263dsp_init_cuda(c) (h263dsp.c:122-123, after ff_h263dsp_init_x86),
 * ff_mpegvideodsp_init_cuda(c) (mpegvideo.c:274, after ff_mpegvideodsp_init(&s->mdsp)) */
void all_hooks_take_the_reference_types(IDCTDSPContext *a, FDCTDSPContext *b, BlockDSPContext *c, MECmpContext *d, H264DSPContext *e,
                                        H264QpelContext *f, H264ChromaContext *g, H264PredContext *h, HpelDSPContext *i,
                                        PixblockDSPContext *j, QpelDSPContext *k, FFTContext *l, H263DSPContext *m, MpegVideoDSPContext *n,
                                        AVCodecContext *avctx)
{
    ff_idctdsp_init_cuda_hook(a, avctx, avctx->bits_per_raw_sample > 8);
    ff_xvid_idct_init_cuda_hook(a, avctx);
    ff_fdctdsp_init_cuda_hook(b, avctx, avctx->bits_per_raw_sample > 8);
    ff_blockdsp_init_cuda(c);
    ff_me_cmp_init_cuda(d);
    ff_h264dsp_init_cuda(e, 8, 1);
    ff_h264qpel_init_cuda(f, 8);
    ff_h264chroma_init_cuda(g, 8);
    ff_h264_pred_init_cuda(h, AV_CODEC_ID_H264, 8, 1);
    ff_hpeldsp_init_cuda(i, avctx->flags);
    ff_pixblockdsp_init_cuda_hook(j, avctx, avctx->bits_per_raw_sample > 8);
    ff_qpeldsp_init_cuda(k);
    ff_fft_init_cuda(l);
    ff_mdct_init_cuda(l);
    ff_h263dsp_init_cuda(m);
    ff_mpegvideodsp_init_cuda(n);
}

/* ---- MECmpContext.quant_psnr / bit / rd (INTEGRATION.md section 2a): called from ff_mpv_encode_init() after the quantiser, the matrices and the
 *      codec's VLC length tables are in place (mpegvideo_enc.c:742-849).  The view holds pointers INTO the context, so the slots follow
 *      qscale / mb_intra as the macroblock loop changes them. ---- */
#include "libavcodec/dct.h"
#include "libavcodec/mpegvideo.h"
typedef struct FFMECmpEncView {
    const int *qscale, *y_dc_scale, *h263_aic, *intra_quant_bias, *inter_quant_bias, *ac_esc_length;
    int *mb_intra, *block_last_index;
    int (*const *q_intra_matrix)[64], (*const *q_inter_matrix)[64];
    const uint16_t *intra_matrix, *inter_matrix;
    const uint8_t *scantable;
    uint8_t *const *intra_ac_vlc_length, *const *intra_ac_vlc_last_length, *const *inter_ac_vlc_length, *const *inter_ac_vlc_last_length;
    const uint8_t *const *luma_dc_vlc_length;
    int fdct, dequant, idct_perm_none, plain_quantiser;
} FFMECmpEncView;
int ff_me_cmp_enc_init_cuda(MECmpContext *c, struct MpegEncContext *s, const FFMECmpEncView *view);
/* the quantiser hook: s->dct_quantize / s->fast_dct_quantize (mpegvideo_enc.c:741, :773-779) */
typedef struct FFMpvQuantView {
    const int *mb_intra, *y_dc_scale, *c_dc_scale, *h263_aic;
    const unsigned *lambda2;
    const int *intra_quant_bias, *inter_quant_bias, *ac_esc_length, *min_qcoeff, *max_qcoeff;
    int (*const *q_intra_matrix)[64], (*const *q_inter_matrix)[64];
    const uint16_t *intra_matrix, *inter_matrix;
    const uint8_t *scantable;
    uint8_t *const *intra_ac_vlc_length, *const *intra_ac_vlc_last_length, *const *inter_ac_vlc_length, *const *inter_ac_vlc_last_length;
    int (*const *dct_error_sum)[64];
    uint16_t (*const *dct_offset)[64];
    int *dct_count, *coded_score;
    int (**dct_quantize)(struct MpegEncContext *, int16_t *, int, int, int *);
    int (**fast_dct_quantize)(struct MpegEncContext *, int16_t *, int, int, int *);
    int fdct, out_format, mpeg_quant, idct_perm_none, quantizer_noise_shaping, slice_context_count;
} FFMpvQuantView;
int ff_mpv_quantize_init_cuda(struct MpegEncContext *s, const FFMpvQuantView *view, int trellis);
int ff_mpv_encode_init_cuda(MpegEncContext *s)
{
    FFMECmpEncView v = {
        .qscale = &s->qscale, .y_dc_scale = &s->y_dc_scale, .h263_aic = &s->h263_aic,
        .intra_quant_bias = &s->intra_quant_bias, .inter_quant_bias = &s->inter_quant_bias, .ac_esc_length = &s->ac_esc_length,
        .mb_intra = &s->mb_intra, .block_last_index = s->block_last_index,
        .q_intra_matrix = &s->q_intra_matrix, .q_inter_matrix = &s->q_inter_matrix,
        .intra_matrix = s->intra_matrix, .inter_matrix = s->inter_matrix, .scantable = s->intra_scantable.scantable,
        .intra_ac_vlc_length = &s->intra_ac_vlc_length, .intra_ac_vlc_last_length = &s->intra_ac_vlc_last_length,
        .inter_ac_vlc_length = &s->inter_ac_vlc_length, .inter_ac_vlc_last_length = &s->inter_ac_vlc_last_length,
        .luma_dc_vlc_length = (const uint8_t *const *)&s->luma_dc_vlc_length,
        .fdct = s->fdsp.fdct == ff_fdct_ifast ? 2 : s->fdsp.fdct == ff_jpeg_fdct_islow_8 ? 0 : s->fdsp.fdct == ff_faandct ? 6 : -1,
        .dequant = s->dct_unquantize_inter == s->dct_unquantize_h263_inter ? 3 :
                   s->dct_unquantize_inter == s->dct_unquantize_mpeg2_inter ? 1 + !!(s->avctx->flags & AV_CODEC_FLAG_BITEXACT) : 0,
        .idct_perm_none = s->idsp.perm_type == FF_IDCT_PERM_NONE,
        .plain_quantiser = s->fast_dct_quantize == ff_dct_quantize_c && !s->dct_error_sum,
    };
    const int r = ff_me_cmp_enc_init_cuda(&s->mecc, s, &v);      /* -1: the C functions ff_me_cmp_init() installed stay */
    /* after the metrics, which must still see fast_dct_quantize == ff_dct_quantize_c; the FFMpvQuantView pointers are the same fields */
    const FFMpvQuantView q = {
        .mb_intra = &s->mb_intra, .y_dc_scale = &s->y_dc_scale, .c_dc_scale = &s->c_dc_scale, .h263_aic = &s->h263_aic,
        .lambda2 = &s->lambda2, .intra_quant_bias = &s->intra_quant_bias, .inter_quant_bias = &s->inter_quant_bias,
        .ac_esc_length = &s->ac_esc_length, .min_qcoeff = &s->min_qcoeff, .max_qcoeff = &s->max_qcoeff,
        .q_intra_matrix = &s->q_intra_matrix, .q_inter_matrix = &s->q_inter_matrix,
        .intra_matrix = s->intra_matrix, .inter_matrix = s->inter_matrix, .scantable = s->intra_scantable.scantable,
        .intra_ac_vlc_length = &s->intra_ac_vlc_length, .intra_ac_vlc_last_length = &s->intra_ac_vlc_last_length,
        .inter_ac_vlc_length = &s->inter_ac_vlc_length, .inter_ac_vlc_last_length = &s->inter_ac_vlc_last_length,
        .dct_error_sum = &s->dct_error_sum, .dct_offset = &s->dct_offset, .dct_count = s->dct_count, .coded_score = s->coded_score,
        .dct_quantize = &s->dct_quantize, .fast_dct_quantize = &s->fast_dct_quantize,
        .fdct = v.fdct, .out_format = s->out_format, .mpeg_quant = s->mpeg_quant,
        .idct_perm_none = s->idsp.perm_type == FF_IDCT_PERM_NONE,
        .quantizer_noise_shaping = s->quantizer_noise_shaping,
        .slice_context_count = s->slice_context_count,           /* > 1 (slice threads): refused, the C quantisers stay */
    };
    ff_mpv_quantize_init_cuda(s, &q, s->avctx->trellis);          /* -1: ff_dct_quantize_c / dct_quantize_trellis_c stay */
    return r;
}

/* ---- libswscale (INTEGRATION.md section 4): the whole-frame SwsFunc and the per-line slots ---- */
static int swscale_cuda(SwsContext *c, const uint8_t *src[], int srcStride[], int srcSliceY, int srcSliceH, uint8_t *dst[], int dstStride[])
{
    SwsContextCUDA *cuda = (SwsContextCUDA *)c->formatConvBuffer;         /* stands for the `cuda` field a maintainer adds to SwsContext */
    return sws_scale_cuda(cuda, (const uint8_t *const *)src, srcStride, srcSliceY, srcSliceH, dst, dstStride);
}
SwsFunc ff_getSwsFunc_cuda(SwsContext *c, SwsContextCUDA **cuda_field)      /* called from ff_getSwsFunc(), swscale.c:773-783 */
{
    SwsLineSlotsCUDA t;
    *cuda_field = sws_getContext_cuda(c->srcW, c->srcH, c->srcFormat, c->dstW, c->dstH, c->dstFormat, c->flags, NULL, NULL, c->param);
    if (!*cuda_field) return NULL;                                      /* not taken over: the C path stays installed */
    if (!ff_sws_init_swscale_cuda(c, *cuda_field, &t)) {                 /* callers that keep the reference's line scheduler swscale() */
        c->hyScale = t.hyScale;           c->hcScale = t.hcScale;
        c->hyscale_fast = t.hyscale_fast; c->hcscale_fast = t.hcscale_fast;
        c->yuv2plane1 = t.yuv2plane1;     c->yuv2planeX = t.yuv2planeX;   c->yuv2nv12cX = t.yuv2nv12cX;
        c->yuv2packed1 = t.yuv2packed1;   c->yuv2packed2 = t.yuv2packed2; c->yuv2packedX = t.yuv2packedX;
        c->lumConvertRange = t.lumConvertRange; c->chrConvertRange = t.chrConvertRange;
    }
    return swscale_cuda;                                                /* whole frames: one call, no per-line round trips */
}
