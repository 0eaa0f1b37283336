/*
 * oracle/refbuild/refapi_prores.c -- TEST INFRASTRUCTURE, NOT PRODUCT.
 *
 * The reference's ProRes decoder and encoder.  This unit #includes libavcodec/proresdec.c and libavcodec/proresenc.c (UNMODIFIED, read in
 * place; the encoder's two struct names are renamed so that both fit in one unit) and prores.mk compiles it with hidden visibility, so only
 * the ref_prores_* functions below leave oracle/_ref/libproresref.so.  proresdsp.c, simple_idct.c and proresdata.c are compiled beside it
 * with CONFIG_PRORES_DECODER / CONFIG_PRORES_ENCODER set.  The glue the two codecs need from the rest of libavcodec (ff_get_buffer,
 * ff_alloc_packet, av_grow_packet, avpriv_request_sample, a serial execute / execute2) is below; it computes nothing.
 *
 *   ref_prores_idct_put   ProresDSPContext.idct_put as ff_proresdsp_init installs it (prores_idct_put_c)
 *   ref_prores_dsp_init   ff_proresdsp_init on a caller's context
 *   ref_prores_abi        sizeof / offsetof of ProresDSPContext
 *   ref_prores_encode     one frame of planes the caller supplies (yuv422p10 / yuv444p10 / yuva444p10, progressive or interlaced) at a
 *                         profile, through encode_init / encode_frame
 *   ref_prores_decode     one frame through decode_init / decode_frame into planes the caller supplies, recording every idct_put call
 *                         (the coefficients before the call, the matrix, the destination) and each picture's slice table
 */
#include <pthread.h>

#include "libavcodec/proresdec.c"
#undef MAX_PADDING
#define ProresContext ProresEncContext
#define ProresThreadData ProresEncThreadData
#include "libavcodec/proresenc.c"
#undef ProresContext
#undef ProresThreadData

#define EXPORT __attribute__((visibility("default")))

/* ---- glue ---------------------------------------------------------------------------------------------------------------------------- */
static uint8_t *g_planes[4];
static int g_linesize[4];

int ff_get_buffer(AVCodecContext *avctx, AVFrame *frame, int flags)
{
    const int alpha = !!(av_pix_fmt_desc_get(avctx->pix_fmt)->flags & AV_PIX_FMT_FLAG_ALPHA);
    (void)flags;
    for (int i = 0; i < 4; i++) {
        frame->data[i] = i < 3 || alpha ? g_planes[i] : NULL;
        frame->linesize[i] = i < 3 || alpha ? g_linesize[i] : 0;
    }
    frame->width = avctx->width; frame->height = avctx->height; frame->format = avctx->pix_fmt;
    return 0;
}
int ff_alloc_packet(AVPacket *avpkt, int size)
{
    avpkt->data = av_mallocz(size + AV_INPUT_BUFFER_PADDING_SIZE);
    avpkt->size = size;
    return avpkt->data ? 0 : AVERROR(ENOMEM);
}
int av_grow_packet(AVPacket *pkt, int grow_by)
{
    uint8_t *p = av_realloc(pkt->data, pkt->size + grow_by + AV_INPUT_BUFFER_PADDING_SIZE);
    if (!p) return AVERROR(ENOMEM);
    memset(p + pkt->size, 0, grow_by + AV_INPUT_BUFFER_PADDING_SIZE);
    pkt->data = p; pkt->size += grow_by;
    return 0;
}
void avpriv_request_sample(void *avc, const char *msg, ...) { (void)avc; (void)msg; }

static int serial_execute2(AVCodecContext *c, int (*func)(AVCodecContext *c2, void *arg2, int jobnr, int threadnr), void *arg2, int *ret,
                           int count)
{
    for (int i = 0; i < count; i++) {
        const int r = func(c, arg2, i, 0);
        if (ret) ret[i] = r;
    }
    return 0;
}

/* ---- the recorder -------------------------------------------------------------------------------------------------------------------- */
typedef struct RefProresRec {
    int32_t cap_blocks, cap_slices;
    int16_t *blocks, *qmat;            /* cap_blocks * 64 each: the coefficients handed to idct_put, the matrix */
    uint64_t *dst;                     /* cap_blocks: the destination pointer */
    uint32_t *slice_first;             /* cap_slices: first block of the slice, counted from its picture's first block */
    uint16_t *slice_sf;                /* cap_slices */
    int32_t n_blocks, n_slices, n_pics, overflow;
    int32_t pic_first_block[2], pic_first_slice[2], pic_n_slices[2], pic_num[2];
    int32_t frame_type, chroma_factor, mb_width, mb_height, slice_width_factor, alpha_info;
    uint8_t qmat_luma[64], qmat_chroma[64];
} RefProresRec;

static RefProresRec *g_rec;
static void (*g_idct_put)(uint16_t *out, ptrdiff_t linesize, int16_t *block, const int16_t *qmat);

static void record_idct_put(uint16_t *out, ptrdiff_t linesize, int16_t *block, const int16_t *qmat)
{
    RefProresRec *r = g_rec;
    if (r->n_blocks < r->cap_blocks) {
        memcpy(r->blocks + 64 * (size_t)r->n_blocks, block, 128);
        memcpy(r->qmat + 64 * (size_t)r->n_blocks, qmat, 128);
        r->dst[r->n_blocks] = (uint64_t)(uintptr_t)out;
    } else r->overflow = 1;
    r->n_blocks++;
    g_idct_put(out, linesize, block, qmat);
}

/* decode_picture's avctx->execute: the slices in order, each one's first block and scale factor recorded */
static int recording_execute(AVCodecContext *c, int (*func)(AVCodecContext *c2, void *arg2), void *arg2, int *ret, int count, int size)
{
    ProresContext *ctx = c->priv_data;
    RefProresRec *r = g_rec;
    const int p = r->n_pics < 2 ? r->n_pics : 1;
    r->pic_first_block[p] = r->n_blocks; r->pic_first_slice[p] = r->n_slices; r->pic_n_slices[p] = count; r->pic_num[p] = ctx->pic_num;
    r->mb_width = ctx->num_x_mbs; r->mb_height = ctx->num_y_mbs; r->slice_width_factor = ctx->slice_width_factor;
    for (int i = 0; i < count; i++) {
        ProresThreadData *td = (ProresThreadData *)((uint8_t *)arg2 + (size_t)i * size);
        const int first = r->n_blocks - r->pic_first_block[p];
        const int rc = func(c, td);
        if (ret) ret[i] = rc;
        if (r->n_slices < r->cap_slices) {
            r->slice_first[r->n_slices] = (uint32_t)first;
            r->slice_sf[r->n_slices] = (uint16_t)td->prev_slice_sf;        /* decode_slice leaves the slice's sf there */
        } else r->overflow = 1;
        r->n_slices++;
    }
    r->n_pics++;
    return 0;
}

/* ---- exports ------------------------------------------------------------------------------------------------------------------------- */
EXPORT void ref_prores_idct_put(uint16_t *out, ptrdiff_t linesize, int16_t *block, const int16_t *qmat)
{
    ProresDSPContext dsp;
    ff_proresdsp_init(&dsp);
    dsp.idct_put(out, linesize, block, qmat);
}

EXPORT void ref_prores_dsp_init(ProresDSPContext *dsp) { ff_proresdsp_init(dsp); }

/* sizeof, offsetof idct_permutation_type, idct_permutation, idct_put */
EXPORT void ref_prores_abi(long out[4])
{
    out[0] = sizeof(ProresDSPContext); out[1] = offsetof(ProresDSPContext, idct_permutation_type);
    out[2] = offsetof(ProresDSPContext, idct_permutation); out[3] = offsetof(ProresDSPContext, idct_put);
}

/* fmt 0 yuv422p10, 1 yuv444p10, 2 yuva444p10; interlaced 0 progressive, 1 top field first, 2 bottom field first; profile 0..4.  Returns the
 * packet size written to out (at most cap), or a negative error. */
EXPORT int ref_prores_encode(int fmt, int width, int height, int interlaced, int profile, uint8_t *const planes[4], const int linesize[4],
                             uint8_t *out, int cap)
{
    static const enum AVPixelFormat fmts[3] = { AV_PIX_FMT_YUV422P10, AV_PIX_FMT_YUV444P10, AV_PIX_FMT_YUVA444P10 };
    if (fmt < 0 || fmt > 2 || interlaced < 0 || interlaced > 2 || profile < 0 || profile > 4) return -1;
    AVCodecContext *avctx = av_mallocz(sizeof(*avctx));
    ProresEncContext *ctx = av_mallocz(sizeof(*ctx));
    AVFrame *frame = av_frame_alloc();
    AVPacket pkt = { 0 };
    int got = 0, rc = -1;
    if (!avctx || !ctx || !frame) goto done;
    av_set_cpu_flags_mask(0);
    ctx->class = &proresenc_class;
    av_opt_set_defaults(ctx);
    ctx->profile = profile;
    avctx->priv_data = ctx;
    avctx->width = width; avctx->height = height; avctx->pix_fmt = fmts[fmt];
    avctx->thread_count = 1;
    avctx->execute2 = serial_execute2;
    avctx->flags = interlaced ? AV_CODEC_FLAG_INTERLACED_DCT : 0;
    avctx->time_base = (AVRational){ 1, 25 };
#if FF_API_CODED_FRAME
    avctx->coded_frame = av_frame_alloc();
#endif
    if (encode_init(avctx) < 0) goto done;
    for (int i = 0; i < 4; i++) { frame->data[i] = planes[i]; frame->linesize[i] = linesize[i]; }
    frame->width = width; frame->height = height; frame->format = avctx->pix_fmt;
    frame->interlaced_frame = !!interlaced; frame->top_field_first = interlaced == 1;
    if (encode_frame(avctx, &pkt, frame, &got) < 0 || !got) goto close;
    rc = pkt.size <= cap ? pkt.size : -2;
    if (rc > 0) memcpy(out, pkt.data, pkt.size);
close:
    encode_close(avctx);
done:
    av_free(pkt.data);
#if FF_API_CODED_FRAME
    if (avctx) av_frame_free(&avctx->coded_frame);
#endif
    av_frame_free(&frame);
    av_free(ctx);
    av_free(avctx);
    return rc;
}

/* Decodes one packet into planes[0..3] (planes[3] is used only when the stream carries alpha) and fills *rec.  Returns decode_frame's
 * result (the packet size) or a negative error. */
EXPORT int ref_prores_decode(const uint8_t *data, int size, int width, int height, uint8_t *const planes[4], const int linesize[4],
                             RefProresRec *rec)
{
    AVCodecContext *avctx = av_mallocz(sizeof(*avctx));
    ProresContext *ctx = av_mallocz(sizeof(*ctx));
    AVFrame *frame = av_frame_alloc();
    uint8_t *buf = av_mallocz(size + AV_INPUT_BUFFER_PADDING_SIZE);
    AVPacket pkt = { 0 };
    int got = 0, rc = -1;
    if (!avctx || !ctx || !frame || !buf) goto done;
    av_set_cpu_flags_mask(0);
    memcpy(buf, data, size);
    pkt.data = buf; pkt.size = size;
    avctx->priv_data = ctx;
    avctx->width = width; avctx->height = height;
    avctx->thread_count = 1;
    avctx->execute = recording_execute;
    for (int i = 0; i < 4; i++) { g_planes[i] = planes[i]; g_linesize[i] = linesize[i]; }
    if (decode_init(avctx) < 0) goto done;
    rec->n_blocks = rec->n_slices = rec->n_pics = rec->overflow = 0;
    g_rec = rec;
    g_idct_put = ctx->dsp.idct_put;
    ctx->dsp.idct_put = record_idct_put;
    rc = decode_frame(avctx, frame, &got, &pkt);
    rec->frame_type = ctx->frame_type; rec->chroma_factor = ctx->chroma_factor; rec->alpha_info = ctx->alpha_info;
    memcpy(rec->qmat_luma, ctx->qmat_luma, 64); memcpy(rec->qmat_chroma, ctx->qmat_chroma, 64);
    decode_close(avctx);
    g_rec = NULL;
done:
    av_frame_free(&frame);
    av_free(buf);
    av_free(ctx);
    av_free(avctx);
    return rc;
}

/* TIMING ONLY (tools/prores_bench.py): prores_idct_put_c over n blocks on `threads` host threads; block i with matrix qidx[i] into
 * frame + dst_off[i] at `linesize` bytes */
typedef struct PutJob {
    int16_t *blocks; const int16_t *qmats; const uint32_t *qidx; uint8_t *frame; const uint32_t *dst_off; ptrdiff_t linesize; size_t lo, hi;
} PutJob;
static void *put_range(void *arg)
{
    PutJob *j = arg;
    ProresDSPContext dsp;
    ff_proresdsp_init(&dsp);
    for (size_t i = j->lo; i < j->hi; i++)
        dsp.idct_put((uint16_t *)(j->frame + j->dst_off[i]), j->linesize, j->blocks + 64 * i, j->qmats + 64 * (size_t)j->qidx[i]);
    return NULL;
}
EXPORT int ref_prores_idct_put_batch(int16_t *blocks, const int16_t *qmats, const uint32_t *qidx, uint8_t *frame, const uint32_t *dst_off,
                                     ptrdiff_t linesize, size_t n, int threads)
{
    pthread_t th[256];
    PutJob jobs[256];
    if (threads < 1) threads = 1;
    if (threads > 256) threads = 256;
    for (int t = 0; t < threads; t++) {
        jobs[t] = (PutJob){ blocks, qmats, qidx, frame, dst_off, linesize, n * t / threads, n * (t + 1) / threads };
        if (pthread_create(&th[t], NULL, put_range, &jobs[t])) return -1;
    }
    for (int t = 0; t < threads; t++) pthread_join(th[t], NULL);
    return 0;
}
