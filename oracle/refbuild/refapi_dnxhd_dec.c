/*
 * oracle/refbuild/refapi_dnxhd_dec.c -- TEST INFRASTRUCTURE, NOT PRODUCT.
 *
 * The reference's VC-3 / DNxHD decoder.  This unit #includes libavcodec/dnxhddec.c (UNMODIFIED, read in place) and dnxhd_dec.mk compiles
 * it with hidden visibility beside bitstream.c and dnxhddata.c, so only the ref_dnxhd_* functions below leave
 * oracle/_ref/libdnxhddecref.so.  Every packet goes through a fresh decoder context, from a copy followed by the zeroed
 * AV_INPUT_BUFFER_PADDING_SIZE bytes a real packet carries.  The shared configuration turns CONFIG_SAFE_BITSTREAM_READER off; the
 * reference's own configure turns it on, and only the checked reader keeps a row that runs off the packet inside the padding, so this unit
 * asks get_bits.h for the checked reader.
 *
 *   ref_dnxhd_decode         one packet into the caller's planes (pre-filled with a sentinel by the caller): the return value and what the
 *                            context reports, and how many "ac tex damaged" messages the decoder logged
 *   ref_dnxhd_cid_table      ff_dnxhd_cid_table and its length
 *   ref_dnxhd_pix_fmts       AV_PIX_FMT_YUV422P, AV_PIX_FMT_YUV422P10 and AV_PIX_FMT_YUV444P10 as this build numbers them
 *   ref_dnxhd_decode_frames  TIMING ONLY: many packets on host threads, one decoder context per thread
 */
#include <pthread.h>
#include <string.h>

#define UNCHECKED_BITSTREAM_READER 0
#include "libavcodec/dnxhddec.c"
#include "libavutil/log.h"

#define EXPORT __attribute__((visibility("default")))

/* ---- glue ---------------------------------------------------------------------------------------------------------------------------- */
/* get_buffer: the caller's planes; refused (ENOMEM) when the frame the decoder asks for does not fit them */
static __thread uint8_t *g_planes[3];
static __thread int g_linesize[3], g_lines, g_get_buffer_calls;
int ff_thread_get_buffer(AVCodecContext *avctx, ThreadFrame *f, int flags)
{
    (void)flags;
    const int bpp = avctx->pix_fmt == AV_PIX_FMT_YUV422P ? 1 : 2, cw = avctx->pix_fmt == AV_PIX_FMT_YUV444P10 ? avctx->width : avctx->width / 2;
    g_get_buffer_calls++;
    if (avctx->width * bpp > g_linesize[0] || cw * bpp > g_linesize[1] || cw * bpp > g_linesize[2] || avctx->height > g_lines)
        return AVERROR(ENOMEM);
    for (int p = 0; p < 3; p++) { f->f->data[p] = g_planes[p]; f->f->linesize[p] = g_linesize[p]; }
    f->f->width = avctx->width; f->f->height = avctx->height; f->f->format = avctx->pix_fmt;
    return 0;
}

int ff_set_dimensions(AVCodecContext *s, int width, int height)
{
    const int ret = av_image_check_size(width, height, 0, s);
    if (ret < 0) width = height = 0;
    s->width = s->coded_width = width;
    s->height = s->coded_height = height;
    return ret;
}

static __thread int g_damaged;
static void count_log(void *avcl, int level, const char *fmt, va_list vl)
{
    (void)avcl; (void)level; (void)vl;
    if (strstr(fmt, "ac tex damaged")) g_damaged++;
}

/* info[0..10] = return value, got_frame, ctx->cid, width, height, pix_fmt, interlaced_frame, top_field_first, sar num, sar den,
 * get_buffer calls; *damaged = the "ac tex damaged" messages logged */
static int decode_one(const uint8_t *pkt, int size, int gray, uint8_t *const planes[3], const int linesize[3], int lines, int32_t *info,
                      int *damaged)
{
    AVCodecContext *avctx = av_mallocz(sizeof(*avctx));
    DNXHDContext *ctx = av_mallocz(sizeof(*ctx));
    AVFrame *frame = av_frame_alloc();
    uint8_t *buf = av_mallocz((size > 0 ? size : 0) + AV_INPUT_BUFFER_PADDING_SIZE);
    int got = 0, ret = -1;
    if (avctx && ctx && frame && buf) {
        memcpy(buf, pkt, size > 0 ? size : 0);
        avctx->priv_data = ctx;
        avctx->flags = gray ? AV_CODEC_FLAG_GRAY : 0;
        avctx->sample_aspect_ratio = (AVRational){ 0, 1 };
        for (int p = 0; p < 3; p++) { g_planes[p] = planes[p]; g_linesize[p] = linesize[p]; }
        g_lines = lines; g_damaged = 0; g_get_buffer_calls = 0;
        AVPacket avpkt = { 0 };
        avpkt.data = buf; avpkt.size = size;
        dnxhd_decode_init(avctx);
        ret = dnxhd_decode_frame(avctx, frame, &got, &avpkt);
        if (info) {
            const int32_t v[11] = { ret, got, ctx->cid, avctx->width, avctx->height, avctx->pix_fmt, frame->interlaced_frame,
                                    frame->top_field_first, avctx->sample_aspect_ratio.num, avctx->sample_aspect_ratio.den, g_get_buffer_calls };
            memcpy(info, v, sizeof(v));
        }
        if (damaged) *damaged = g_damaged;
        dnxhd_decode_close(avctx);
    }
    av_free(buf);
    av_frame_free(&frame);
    av_free(ctx);
    av_free(avctx);
    return ret;
}

EXPORT int ref_dnxhd_decode(const uint8_t *pkt, int size, int gray, uint8_t *const *planes, const int *linesize, int lines, int32_t *info,
                            int *damaged)
{
    av_log_set_callback(count_log);
    const int ret = decode_one(pkt, size, gray, planes, linesize, lines, info, damaged);
    av_log_set_callback(av_log_default_callback);
    return ret;
}

EXPORT const CIDEntry *ref_dnxhd_cid_table(int *n)
{
    int last = -1;
    for (int cid = 1; cid < 4096; cid++) {
        const int i = ff_dnxhd_get_cid_table(cid);
        if (i > last) last = i;
    }
    *n = last + 1;
    return ff_dnxhd_cid_table;
}

EXPORT void ref_dnxhd_pix_fmts(int32_t *out)
{
    out[0] = AV_PIX_FMT_YUV422P; out[1] = AV_PIX_FMT_YUV422P10; out[2] = AV_PIX_FMT_YUV444P10;
}

/* TIMING ONLY (tools/dnxhd_dec_bench.py): packets lo..hi of n on one thread, each into its own planes (3 per packet) */
typedef struct DecJob { const uint8_t *const *pkts; const int *sizes; uint8_t *const *planes; const int *linesizes; int lines, lo, hi; } DecJob;
static void *decode_range(void *arg)
{
    DecJob *j = arg;
    for (int k = j->lo; k < j->hi; k++) decode_one(j->pkts[k], j->sizes[k], 0, j->planes + 3 * k, j->linesizes + 3 * k, j->lines, NULL, NULL);
    return NULL;
}
EXPORT int ref_dnxhd_decode_frames(const uint8_t *const *pkts, const int *sizes, int n, uint8_t *const *planes, const int *linesizes, int lines,
                                   int threads)
{
    pthread_t th[256];
    DecJob jobs[256];
    if (threads < 1) threads = 1;
    if (threads > 256) threads = 256;
    if (threads > n) threads = n;
    av_log_set_level(AV_LOG_QUIET);
    for (int t = 0; t < threads; t++) {
        jobs[t] = (DecJob){ pkts, sizes, planes, linesizes, lines, n * t / threads, n * (t + 1) / threads };
        if (pthread_create(&th[t], NULL, decode_range, &jobs[t])) return -1;
    }
    for (int t = 0; t < threads; t++) pthread_join(th[t], NULL);
    return 0;
}
