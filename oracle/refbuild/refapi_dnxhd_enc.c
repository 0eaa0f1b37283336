/*
 * oracle/refbuild/refapi_dnxhd_enc.c -- TEST INFRASTRUCTURE, NOT PRODUCT.
 *
 * The reference's VC-3 / DNxHD encoder with every option it has.  This unit #includes libavcodec/dnxhdenc.c (UNMODIFIED, read in place)
 * and dnxhd_enc.mk compiles it with hidden visibility beside dnxhddata.c, so only the ref_dnxhd_* functions below leave
 * oracle/_ref/libdnxhdencref.so.  libavref.so provides the DSP inits, the quantiser and the option / frame helpers; it exports
 * ff_alloc_packet and av_packet_new_side_data only as aborting stand-ins, so this unit defines working ones, which bind locally.  The
 * encoder runs its slices through a serial execute2, and its CID lookup returns the requested CID (see glue_find_cid).  Opening
 * a context fills ff_square_tab as avcodec_init does (the variance pass of the fast rate control reads it through pix_norm1).
 *
 *   ref_dnxhd_encode_seq     frames through one context: each packet, and the return value, qscale, lambda and quality after each
 *   ref_dnxhd_cid_entry      &ff_dnxhd_cid_table[i] of a CID (the entry a context's cid_table points at)
 *   ref_dnxhd_vlc            the context's vlc_codes / vlc_bits / run_codes / run_bits after encode_init
 *   ref_dnxhd_cid_layout     sizeof(CIDEntry) and the offset of each of its fields
 *   ref_dnxhd_encode_frames  TIMING ONLY: many frames on host threads, one encoder context per thread
 */
#include <pthread.h>
#include <stddef.h>

/* ff_dnxhd_find_cid as compiled here returns the first CID of the frame size whatever the bit rate (its loop over bit_rates runs past
 * the array, and the compiler assumes it stops inside), so 1238, 1243, 1252, 1253 and 1256 cannot be chosen through bit_rate.  The
 * encoder's one call of it goes to glue_find_cid, which returns the CID the caller asked for. */
#define ff_dnxhd_find_cid glue_find_cid
#include "libavcodec/dnxhdenc.c"
#undef ff_dnxhd_find_cid

#define EXPORT __attribute__((visibility("default")))

/* ---- glue ---------------------------------------------------------------------------------------------------------------------------- */
void ff_dnxhdenc_init_x86(DNXHDEncContext *c) { (void)c; }      /* ARCH_X86 is 0 in this configuration: never called */

int ff_alloc_packet(AVPacket *avpkt, int size)
{
    avpkt->data = av_mallocz(size + AV_INPUT_BUFFER_PADDING_SIZE);
    avpkt->size = size;
    return avpkt->data ? 0 : AVERROR(ENOMEM);
}
static __thread int g_quality[4];
uint8_t *av_packet_new_side_data(AVPacket *pkt, enum AVPacketSideDataType type, int size)
{
    (void)pkt; (void)type;
    return size <= (int)sizeof(g_quality) ? (uint8_t *)g_quality : NULL;
}

static __thread int g_want_cid;
int glue_find_cid(AVCodecContext *avctx, int bit_depth)
{
    const int index = ff_dnxhd_get_cid_table(g_want_cid);
    return index >= 0 && ff_dnxhd_cid_table[index].bit_depth == bit_depth ? g_want_cid : 0;
}

static int serial_execute2(AVCodecContext *c, int (*func)(AVCodecContext *c2, void *arg2, int jobnr, int threadnr), void *arg2, int *ret,
                           int count)
{
    for (int i = 0; i < count; i++) {
        const int r = func(c, arg2, i, 0);
        if (ret) ret[i] = r;
    }
    return 0;
}

/* interlaced 0 progressive, 1 top field first, 2 bottom field first; mb_decision, qmax, dct_algo as AVCodecContext has them;
 * nitris_compat and ibias as the encoder's private options (ibias 999999 is its default) */
typedef struct RefDnxhdOpts { int32_t cid, interlaced, dct_algo, mb_decision, qmax, nitris_compat, ibias; } RefDnxhdOpts;
typedef struct RefEnc { AVCodecContext *avctx; DNXHDEncContext *ctx; } RefEnc;

static void close_enc(RefEnc *e)
{
    if (e->ctx && e->ctx->cid_table) dnxhd_encode_end(e->avctx);
#if FF_API_CODED_FRAME
    if (e->avctx) av_frame_free(&e->avctx->coded_frame);
#endif
    av_freep(&e->ctx);
    av_freep(&e->avctx);
}

static int open_enc(RefEnc *e, const RefDnxhdOpts *o)
{
    const int index = ff_dnxhd_get_cid_table(o->cid);
    if (index < 0) return -1;
    const CIDEntry *cid = &ff_dnxhd_cid_table[index];
    e->avctx = av_mallocz(sizeof(*e->avctx));
    e->ctx = av_mallocz(sizeof(*e->ctx));
    if (!e->avctx || !e->ctx) return -1;
    av_set_cpu_flags_mask(0);
    ff_me_cmp_init_static();                      /* ff_square_tab, which pix_norm1 reads: avcodec_init fills it in a real program */
    e->ctx->class = &class;
    av_opt_set_defaults(e->ctx);
    e->ctx->nitris_compat = o->nitris_compat;
    e->ctx->intra_quant_bias = o->ibias;
    e->avctx->priv_data = e->ctx;
    e->avctx->width = cid->width; e->avctx->height = cid->height;
    e->avctx->pix_fmt = cid->bit_depth == 10 ? AV_PIX_FMT_YUV422P10 : AV_PIX_FMT_YUV422P;
    e->avctx->flags = cid->interlaced ? AV_CODEC_FLAG_INTERLACED_DCT : 0;
    e->avctx->mb_decision = o->mb_decision;
    e->avctx->qmax = o->qmax;
    e->avctx->dct_algo = o->dct_algo;
    e->avctx->thread_count = 1;
    e->avctx->execute2 = serial_execute2;
    e->avctx->time_base = (AVRational){ 1, 25 };
    e->avctx->bit_rate = (int64_t)cid->bit_rates[0] * 1000000;
    g_want_cid = o->cid;
#if FF_API_CODED_FRAME
    e->avctx->coded_frame = av_frame_alloc();
#endif
    return dnxhd_encode_init(e->avctx) < 0 ? -1 : 0;
}

/* one frame: planes y / u / v with their linesizes; the packet into out (frame_size bytes); rc[0..3] = the return value, ctx->qscale,
 * ctx->lambda, the quality side data (0 when the encode failed) */
static void encode_one(RefEnc *e, const RefDnxhdOpts *o, uint8_t *const planes[3], const int linesize[3], uint8_t *out, int32_t *rc)
{
    AVFrame *frame = av_frame_alloc();
    AVPacket pkt = { 0 };
    int got = 0;
    for (int i = 0; i < 3; i++) { frame->data[i] = planes[i]; frame->linesize[i] = linesize[i]; }
    frame->width = e->avctx->width; frame->height = e->avctx->height; frame->format = e->avctx->pix_fmt;
    frame->interlaced_frame = !!o->interlaced; frame->top_field_first = o->interlaced == 1;
    g_quality[0] = 0;
    rc[0] = dnxhd_encode_picture(e->avctx, &pkt, frame, &got);
    rc[1] = (int32_t)e->ctx->qscale; rc[2] = (int32_t)e->ctx->lambda; rc[3] = rc[0] >= 0 ? g_quality[0] : 0;
    if (rc[0] >= 0 && got) memcpy(out, pkt.data, pkt.size);
    av_free(pkt.data);
    av_frame_free(&frame);
}

/* n frames through one context: planes[3 k + p], linesizes[3 k + p]; packet k at out + k * frame_size; rc[4 k ..].  Returns frame_size,
 * or -1 when encode_init refuses the options */
EXPORT int ref_dnxhd_encode_seq(const RefDnxhdOpts *o, int n, uint8_t *const *planes, const int *linesizes, uint8_t *out, int32_t *rc)
{
    RefEnc e = { 0 };
    int size = -1;
    if (open_enc(&e, o) == 0) {
        size = (int)e.ctx->cid_table->frame_size;
        for (int k = 0; k < n; k++) encode_one(&e, o, planes + 3 * k, linesizes + 3 * k, out + (size_t)k * size, rc + 4 * k);
    }
    close_enc(&e);
    return size;
}

EXPORT const CIDEntry *ref_dnxhd_cid_entry(int cid)
{
    const int index = ff_dnxhd_get_cid_table(cid);
    return index < 0 ? NULL : &ff_dnxhd_cid_table[index];
}

/* after encode_init: vlc_codes / vlc_bits for levels -max_level..max_level - 1 (index (level << 1 | run) + 2 max_level), run_codes /
 * run_bits 0..62.  Returns max_level, or -1 */
EXPORT int ref_dnxhd_vlc(const RefDnxhdOpts *o, uint32_t *codes, uint8_t *bits, uint16_t *run_codes, uint8_t *run_bits)
{
    RefEnc e = { 0 };
    int ml = -1;
    if (open_enc(&e, o) == 0) {
        ml = 1 << (e.ctx->cid_table->bit_depth + 2);
        for (int i = 0; i < 4 * ml; i++) { codes[i] = e.ctx->vlc_codes[i - 2 * ml]; bits[i] = e.ctx->vlc_bits[i - 2 * ml]; }
        for (int i = 0; i < 63; i++) { run_codes[i] = e.ctx->run_codes[i]; run_bits[i] = e.ctx->run_bits[i]; }
    }
    close_enc(&e);
    return ml;
}

/* sizeof(CIDEntry), then the offset of each field in declaration order; returns the count */
EXPORT int ref_dnxhd_cid_layout(int32_t *out)
{
    int n = 0;
    out[n++] = sizeof(CIDEntry);
#define OFF(f) out[n++] = offsetof(CIDEntry, f)
    OFF(cid); OFF(width); OFF(height); OFF(interlaced); OFF(frame_size); OFF(coding_unit_size); OFF(index_bits); OFF(bit_depth);
    OFF(luma_weight); OFF(chroma_weight); OFF(dc_codes); OFF(dc_bits); OFF(ac_codes); OFF(ac_bits); OFF(ac_level); OFF(ac_run_flag);
    OFF(ac_index_flag); OFF(run_codes); OFF(run_bits); OFF(run); OFF(bit_rates);
#undef OFF
    return n;
}

/* TIMING ONLY (tools/dnxhd_enc_bench.py): frames lo..hi of n on one thread, one context; planes / linesizes: 3 per frame */
typedef struct EncJob {
    const RefDnxhdOpts *o; uint8_t *const *planes; const int *linesizes; uint8_t *out; int32_t *rc; int lo, hi;
} EncJob;
static void *encode_range(void *arg)
{
    EncJob *j = arg;
    RefEnc e = { 0 };
    if (open_enc(&e, j->o) == 0)
        for (int k = j->lo; k < j->hi; k++)
            encode_one(&e, j->o, j->planes + 3 * k, j->linesizes + 3 * k, j->out + (size_t)k * e.ctx->cid_table->frame_size, j->rc + 4 * k);
    close_enc(&e);
    return NULL;
}
EXPORT int ref_dnxhd_encode_frames(const RefDnxhdOpts *o, int n, uint8_t *const *planes, const int *linesizes, uint8_t *out, int32_t *rc,
                                   int threads)
{
    pthread_t th[256];
    EncJob jobs[256];
    if (threads < 1) threads = 1;
    if (threads > 256) threads = 256;
    if (threads > n) threads = n;
    for (int k = 0; k < n; k++) rc[4 * k] = -1;
    for (int t = 0; t < threads; t++) {
        jobs[t] = (EncJob){ o, planes, linesizes, out, rc, n * t / threads, n * (t + 1) / threads };
        if (pthread_create(&th[t], NULL, encode_range, &jobs[t])) return -1;
    }
    for (int t = 0; t < threads; t++) pthread_join(th[t], NULL);
    return 0;
}
