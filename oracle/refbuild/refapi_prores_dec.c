/*
 * oracle/refbuild/refapi_prores_dec.c -- TEST INFRASTRUCTURE, NOT PRODUCT.
 *
 * The reference's ProRes decoder with the checked bitstream reader.  This unit #includes libavcodec/proresdec.c (UNMODIFIED, read in
 * place) and prores_dec.mk compiles it with hidden visibility beside prores.mk's proresdsp.c, simple_idct.c and proresdata.c objects, so
 * only the ref_prores_dec_* functions below leave oracle/_ref/libproresdecref.so.  The shared configuration turns
 * CONFIG_SAFE_BITSTREAM_READER off; the reference's own configure turns it on, and only the checked reader clamps a slice plane's reads,
 * so this unit asks get_bits.h for the checked reader.  (libproresref.so keeps the unchecked one for the flush-point tests.)
 *
 * Every packet is decoded from a copy followed by zeroed padding (the reader's 64-bit load at its clamp position touches 9 bytes past a
 * plane that ends the packet; it uses 5 of them), into the caller's planes (pre-filled with a sentinel by the caller), through a serial
 * execute with avcodec_default_execute's semantics (each slice's return value is ignored).
 *
 *   ref_prores_dec_decode         packets 0..n-1 through ONE decoder context in turn (n = 1: a fresh context), each into its own planes,
 *                                 with the context state the probe mirrors
 *   ref_prores_dec_tables         proresdata.c's scans, codebooks and index tables, and FIRST_DC_CB
 *   ref_prores_dec_pix_fmts       AV_PIX_FMT_YUV422P10, YUV444P10, YUVA422P10 and YUVA444P10 as this build numbers them
 *   ref_prores_dec_neg_usr32      NEG_USR32 as this build compiles it (the shift count is a run-time value, as in decode_vlc_codeword)
 *   ref_prores_dec_decode_frames  TIMING ONLY: many packets on host threads, one fresh context per packet
 */
#include <pthread.h>
#include <string.h>

#define UNCHECKED_BITSTREAM_READER 0
#include "libavcodec/proresdec.c"
#include "libavutil/log.h"

#define EXPORT __attribute__((visibility("default")))
#define PADDING 16

/* ---- glue ---------------------------------------------------------------------------------------------------------------------------- */
static __thread uint8_t *const *g_planes;
static __thread const int *g_linesize;
static __thread int g_get_buffer_calls, g_pictures;

int ff_get_buffer(AVCodecContext *avctx, AVFrame *frame, int flags)
{
    const int alpha = avctx->pix_fmt == AV_PIX_FMT_YUVA422P10 || avctx->pix_fmt == AV_PIX_FMT_YUVA444P10;
    (void)flags;
    g_get_buffer_calls++;
    for (int i = 0; i < 4; i++) {
        frame->data[i] = i < 3 || alpha ? g_planes[i] : NULL;
        frame->linesize[i] = i < 3 || alpha ? g_linesize[i] : 0;
    }
    frame->width = avctx->width; frame->height = avctx->height; frame->format = avctx->pix_fmt;
    return 0;
}

/* avcodec_default_execute, counting decode_picture's calls */
static int serial_execute(AVCodecContext *c, int (*func)(AVCodecContext *c2, void *arg2), void *arg, int *ret, int count, int size)
{
    g_pictures++;
    for (int i = 0; i < count; i++) {
        const int r = func(c, (char *)arg + (size_t)i * size);
        if (ret) ret[i] = r;
    }
    return 0;
}

/* info[0..12] per packet: return value, got_frame, pix_fmt, interlaced_frame, top_field_first, color_primaries, color_trc, colorspace,
 * pictures decoded (execute calls), get_buffer calls, frame_type, alpha_info, num_y_mbs */
static void decode_seq(const uint8_t *const *pkts, const int *sizes, int n, int width, int height, uint8_t *const *planes,
                       const int *linesizes, int32_t *info)
{
    AVCodecContext *avctx = av_mallocz(sizeof(*avctx));
    ProresContext *ctx = av_mallocz(sizeof(*ctx));
    if (!avctx || !ctx) goto done;
    avctx->priv_data = ctx;
    avctx->width = width; avctx->height = height;
    avctx->thread_count = 1;
    avctx->execute = serial_execute;
    decode_init(avctx);
    for (int k = 0; k < n; k++) {
        const int size = sizes[k] > 0 ? sizes[k] : 0;
        uint8_t *buf = av_mallocz(size + PADDING);
        AVFrame *frame = av_frame_alloc();
        if (!buf || !frame) { av_free(buf); av_frame_free(&frame); break; }
        memcpy(buf, pkts[k], size);
        AVPacket pkt = { 0 };
        pkt.data = buf; pkt.size = sizes[k];
        g_planes = planes + 4 * k; g_linesize = linesizes + 4 * k;
        g_get_buffer_calls = g_pictures = 0;
        int got = 0;
        const int ret = decode_frame(avctx, frame, &got, &pkt);
        if (info) {
            const int32_t v[13] = { ret, got, avctx->pix_fmt, frame->interlaced_frame, frame->top_field_first, avctx->color_primaries,
                                    avctx->color_trc, avctx->colorspace, g_pictures, g_get_buffer_calls, ctx->frame_type, ctx->alpha_info,
                                    ctx->num_y_mbs };
            memcpy(info + 13 * k, v, sizeof(v));
        }
        av_frame_free(&frame);
        av_free(buf);
    }
    decode_close(avctx);
done:
    av_free(ctx);
    av_free(avctx);
}

/* ---- exports ------------------------------------------------------------------------------------------------------------------------- */
EXPORT void ref_prores_dec_decode(const uint8_t *const *pkts, const int *sizes, int n, int width, int height, uint8_t *const *planes,
                                  const int *linesizes, int32_t *info)
{
    av_log_set_level(AV_LOG_QUIET);
    decode_seq(pkts, sizes, n, width, height, planes, linesizes, info);
}

/* both scans, the DC and AC codebooks, run_to_cb_index, lev_to_cb_index, FIRST_DC_CB; returns the count */
EXPORT int ref_prores_dec_tables(int32_t *out)
{
    int n = 0;
    for (int i = 0; i < 64; i++) out[n++] = ff_prores_progressive_scan[i];
    for (int i = 0; i < 64; i++) out[n++] = ff_prores_interlaced_scan[i];
    for (int i = 0; i < 4; i++) out[n++] = ff_prores_dc_codebook[i];
    for (int i = 0; i < 7; i++) out[n++] = ff_prores_ac_codebook[i];
    for (int i = 0; i < 16; i++) out[n++] = ff_prores_run_to_cb_index[i];
    for (int i = 0; i < 10; i++) out[n++] = ff_prores_lev_to_cb_index[i];
    out[n++] = FIRST_DC_CB;
    return n;
}

EXPORT void ref_prores_dec_pix_fmts(int32_t *out)
{
    out[0] = AV_PIX_FMT_YUV422P10; out[1] = AV_PIX_FMT_YUV444P10; out[2] = AV_PIX_FMT_YUVA422P10; out[3] = AV_PIX_FMT_YUVA444P10;
}

EXPORT uint32_t ref_prores_dec_neg_usr32(uint32_t a, int s) { return NEG_USR32(a, s); }

/* TIMING ONLY (tools/prores_dec_bench.py): packets lo..hi of n on one thread, each through a fresh context into its own planes (4 per
 * packet) */
typedef struct DecJob {
    const uint8_t *const *pkts; const int *sizes; uint8_t *const *planes; const int *linesizes; int width, height, lo, hi;
} DecJob;
static void *decode_range(void *arg)
{
    DecJob *j = arg;
    for (int k = j->lo; k < j->hi; k++)
        decode_seq(j->pkts + k, j->sizes + k, 1, j->width, j->height, j->planes + 4 * k, j->linesizes + 4 * k, NULL);
    return NULL;
}
EXPORT int ref_prores_dec_decode_frames(const uint8_t *const *pkts, const int *sizes, int n, int width, int height, uint8_t *const *planes,
                                        const int *linesizes, int threads)
{
    pthread_t th[256];
    DecJob jobs[256];
    if (threads < 1) threads = 1;
    if (threads > 256) threads = 256;
    if (threads > n) threads = n;
    av_log_set_level(AV_LOG_QUIET);
    for (int t = 0; t < threads; t++) {
        jobs[t] = (DecJob){ pkts, sizes, planes, linesizes, width, height, n * t / threads, n * (t + 1) / threads };
        if (pthread_create(&th[t], NULL, decode_range, &jobs[t])) return -1;
    }
    for (int t = 0; t < threads; t++) pthread_join(th[t], NULL);
    return 0;
}
