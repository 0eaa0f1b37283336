/*
 * oracle/refbuild/refapi_prores_enc.c -- TEST INFRASTRUCTURE, NOT PRODUCT.
 *
 * The reference's ProRes encoder with every option it has.  This unit #includes libavcodec/proresenc.c (UNMODIFIED, read in place) and
 * prores_enc.mk compiles it with hidden visibility, so only the ref_prores_enc* functions below leave oracle/_ref/libproresencref.so.
 * proresdata.c is compiled beside it.  The glue the encoder needs from the rest of libavcodec (ff_alloc_packet, av_grow_packet,
 * avpriv_request_sample, a serial execute2) computes nothing; the execute2 of ref_prores_encode_opts also copies each picture's
 * ctx->slice_q once find_quant_thread has filled it.
 *
 *   ref_prores_encode_opts    one frame through encode_init / encode_frame with every option: the packet and each slice's quantiser
 *   ref_prores_enc_tables     the tables the encoder codes with (proresdata.c and proresenc.c's own)
 *   ref_prores_encode_frames  TIMING ONLY: many frames on host threads, one encoder context per thread
 */
#include <pthread.h>

#include "libavcodec/proresenc.c"

#define EXPORT __attribute__((visibility("default")))

/* ---- glue ---------------------------------------------------------------------------------------------------------------------------- */
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

/* the recording of ref_prores_encode_opts (one thread: the timing export never records) */
static int32_t *g_slice_q;
static int g_cap_q, g_pics;

static int serial_execute2(AVCodecContext *c, int (*func)(AVCodecContext *c2, void *arg2, int jobnr, int threadnr), void *arg2, int *ret,
                           int count)
{
    ProresContext *ctx = c->priv_data;
    for (int i = 0; i < count; i++) {
        const int r = func(c, arg2, i, 0);
        if (ret) ret[i] = r;
    }
    if (g_slice_q) {
        for (int i = 0; i < ctx->slices_per_picture; i++) {
            const int k = g_pics * ctx->slices_per_picture + i;
            if (k < g_cap_q) g_slice_q[k] = ctx->slice_q[i];
        }
        g_pics++;
    }
    return 0;
}

/* fmt 0 yuv422p10, 1 yuv444p10, 2 yuva444p10; interlaced 0 progressive, 1 top field first, 2 bottom field first; the rest as the
 * encoder's options (force_quant q goes in as global_quality = q * FF_QP2LAMBDA) */
typedef struct RefProresEncOpts {
    int32_t fmt, interlaced, profile, mbs_per_slice, bits_per_mb, quant_sel, alpha_bits, force_quant;
    char vendor[4];
    uint8_t color_primaries, color_trc, colorspace, reserved;
} RefProresEncOpts;

typedef struct RefEnc { AVCodecContext *avctx; ProresContext *ctx; } RefEnc;

static void close_enc(RefEnc *e)
{
    if (e->ctx) {
        if (e->ctx->tdata || e->ctx->slice_q) encode_close(e->avctx);
        av_opt_free(e->ctx);
    }
#if FF_API_CODED_FRAME
    if (e->avctx) av_frame_free(&e->avctx->coded_frame);
#endif
    av_freep(&e->ctx);
    av_freep(&e->avctx);
}

static int open_enc(RefEnc *e, const RefProresEncOpts *o, int width, int height)
{
    static const enum AVPixelFormat fmts[3] = { AV_PIX_FMT_YUV422P10, AV_PIX_FMT_YUV444P10, AV_PIX_FMT_YUVA444P10 };
    char vendor[5];
    e->avctx = av_mallocz(sizeof(*e->avctx));
    e->ctx = av_mallocz(sizeof(*e->ctx));
    if (!e->avctx || !e->ctx || o->fmt < 0 || o->fmt > 2 || o->interlaced < 0 || o->interlaced > 2) return -1;
    av_set_cpu_flags_mask(0);
    e->ctx->class = &proresenc_class;
    av_opt_set_defaults(e->ctx);
    e->ctx->profile = o->profile; e->ctx->mbs_per_slice = o->mbs_per_slice; e->ctx->bits_per_mb = o->bits_per_mb;
    e->ctx->quant_sel = o->quant_sel; e->ctx->alpha_bits = o->alpha_bits;
    memcpy(vendor, o->vendor, 4); vendor[4] = 0;
    av_free(e->ctx->vendor);
    e->ctx->vendor = av_strdup(vendor);
    e->avctx->priv_data = e->ctx;
    e->avctx->width = width; e->avctx->height = height; e->avctx->pix_fmt = fmts[o->fmt];
    e->avctx->global_quality = o->force_quant * FF_QP2LAMBDA;
    e->avctx->color_primaries = o->color_primaries; e->avctx->color_trc = o->color_trc; e->avctx->colorspace = o->colorspace;
    e->avctx->thread_count = 1;
    e->avctx->execute2 = serial_execute2;
    e->avctx->flags = o->interlaced ? AV_CODEC_FLAG_INTERLACED_DCT : 0;
    e->avctx->time_base = (AVRational){ 1, 25 };
#if FF_API_CODED_FRAME
    e->avctx->coded_frame = av_frame_alloc();
#endif
    return encode_init(e->avctx) < 0 ? -1 : 0;
}

/* one packet into out (at most cap bytes); cap_q slice quantisers into slice_q (pictures in order, each in raster order).  Returns the
 * packet size, -1 when encode_init refuses the options, -2 when the packet exceeds cap. */
static int encode_one(RefEnc *e, const RefProresEncOpts *o, int width, int height, uint8_t *const planes[4], const int linesize[4],
                      uint8_t *out, int cap)
{
    AVFrame *frame = av_frame_alloc();
    AVPacket pkt = { 0 };
    int got = 0, rc = -1;
    if (!frame) return -1;
    for (int i = 0; i < 4; i++) { frame->data[i] = planes[i]; frame->linesize[i] = linesize[i]; }
    frame->width = width; frame->height = height; frame->format = e->avctx->pix_fmt;
    frame->interlaced_frame = !!o->interlaced; frame->top_field_first = o->interlaced == 1;
    if (encode_frame(e->avctx, &pkt, frame, &got) >= 0 && got) {
        rc = pkt.size <= cap ? pkt.size : -2;
        if (rc > 0) memcpy(out, pkt.data, pkt.size);
    }
    av_free(pkt.data);
    av_frame_free(&frame);
    return rc;
}

EXPORT int ref_prores_encode_opts(const RefProresEncOpts *o, int width, int height, uint8_t *const planes[4], const int linesize[4],
                                  uint8_t *out, int cap, int32_t *slice_q, int cap_q)
{
    RefEnc e = { 0 };
    int rc = -1;
    if (open_enc(&e, o, width, height) == 0) {
        const int n = e.ctx->slices_per_picture * e.ctx->pictures_per_frame;
        for (int i = 0; i < n && i < cap_q; i++) slice_q[i] = e.ctx->force_quant;      /* forced: find_quant_thread never runs */
        g_slice_q = slice_q; g_cap_q = cap_q; g_pics = 0;
        rc = encode_one(&e, o, width, height, planes, linesize, out, cap);
        g_slice_q = NULL;
    }
    close_enc(&e);
    return rc;
}

/* both scans, the DC and AC codebooks, run_to_cb_index, lev_to_cb_index, FIRST_DC_CB, the quantiser matrices, per profile min_quant /
 * max_quant / br_tab[4], prores_mb_limits; returns the count */
EXPORT int ref_prores_enc_tables(int32_t *out)
{
    int n = 0;
    for (int i = 0; i < 64; i++) out[n++] = ff_prores_progressive_scan[i];
    for (int i = 0; i < 64; i++) out[n++] = ff_prores_interlaced_scan[i];
    for (int i = 0; i < 4; i++) out[n++] = ff_prores_dc_codebook[i];
    for (int i = 0; i < 7; i++) out[n++] = ff_prores_ac_codebook[i];
    for (int i = 0; i < 16; i++) out[n++] = ff_prores_run_to_cb_index[i];
    for (int i = 0; i < 10; i++) out[n++] = ff_prores_lev_to_cb_index[i];
    out[n++] = FIRST_DC_CB;
    for (int m = 0; m < 5; m++) for (int i = 0; i < 64; i++) out[n++] = prores_quant_matrices[m][i];
    for (int p = 0; p < 5; p++) {
        out[n++] = prores_profile_info[p].min_quant; out[n++] = prores_profile_info[p].max_quant;
        for (int i = 0; i < 4; i++) out[n++] = prores_profile_info[p].br_tab[i];
    }
    for (int i = 0; i < NUM_MB_LIMITS; i++) out[n++] = prores_mb_limits[i];
    return n;
}

/* TIMING ONLY (tools/prores_enc_bench.py): frames lo..hi of n on one thread, one context; planes: 4 per frame, outs: one per frame */
typedef struct EncJob {
    const RefProresEncOpts *o; int width, height; uint8_t *const *planes; const int *linesize; uint8_t *const *outs; int cap; int32_t *sizes;
    int lo, hi;
} EncJob;
static void *encode_range(void *arg)
{
    EncJob *j = arg;
    RefEnc e = { 0 };
    if (open_enc(&e, j->o, j->width, j->height) == 0)
        for (int k = j->lo; k < j->hi; k++)
            j->sizes[k] = encode_one(&e, j->o, j->width, j->height, j->planes + 4 * k, j->linesize, j->outs[k], j->cap);
    close_enc(&e);
    return NULL;
}
EXPORT int ref_prores_encode_frames(const RefProresEncOpts *o, int width, int height, int n, uint8_t *const *planes, const int linesize[4],
                                    uint8_t *const *outs, int cap, int32_t *sizes, int threads)
{
    pthread_t th[256];
    EncJob jobs[256];
    if (threads < 1) threads = 1;
    if (threads > 256) threads = 256;
    if (threads > n) threads = n;
    for (int k = 0; k < n; k++) sizes[k] = -1;
    for (int t = 0; t < threads; t++) {
        jobs[t] = (EncJob){ o, width, height, planes, linesize, outs, cap, sizes, n * t / threads, n * (t + 1) / threads };
        if (pthread_create(&th[t], NULL, encode_range, &jobs[t])) return -1;
    }
    for (int t = 0; t < threads; t++) pthread_join(th[t], NULL);
    return 0;
}
