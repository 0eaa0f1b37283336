/*
 * oracle/refbuild/refapi_mpvq.c -- TEST INFRASTRUCTURE, NOT PRODUCT.
 *
 * The reference's encoder quantisers.  dct_quantize_trellis_c, denoise_dct_c, clip_coeffs and dct_single_coeff_elimination are static in
 * libavcodec/mpegvideo_enc.c, so this unit #includes that file (UNMODIFIED, read in place) and exports only the ref_mpvq_* wrappers below;
 * Makefile compiles it with hidden visibility, so the file's own external names stay inside oracle/_ref/libmpvqref.so, and links it against
 * libavref.so for everything else (the FDCTs, av_log, the encoder's stubs).
 *
 * ref_mpvq_batch() runs, for every record, what encode_mb_internal (mpegvideo_enc.c:2263-2303) runs for one block on one context:
 *   last = s->dct_quantize(s, s->block[n], n, qscale, &overflow)   (ff_dct_quantize_c, or dct_quantize_trellis_c; denoise_dct_c inside
 *                                                                   when s->dct_error_sum is set)
 *   post: if (overflow) clip_coeffs(...); block_last_index[n] = last; dct_single_coeff_elimination(s, n, threshold) for an inter block
 *         with a threshold (luma for n < 4, chroma for n >= 4)
 * in record order on one context, so the noise-reduction sums are the encoder's sequential ones.  No arithmetic of its own.
 */
#include "libavcodec/mpegvideo_enc.c"

#define EXPORT __attribute__((visibility("default")))

/* include/avdsp_b200.h FFMpvQuantState / FFMpvQuantRecord, same layout */
typedef struct MpvqState {
    int32_t fdct, out_format, mpeg_quant, h263_aic, intra_quant_bias, inter_quant_bias, ac_esc_length, min_qcoeff, max_qcoeff;
    int32_t luma_elim_threshold, chroma_elim_threshold;
    int32_t q_intra_matrix[32][64], q_inter_matrix[32][64];
    uint16_t intra_matrix[64], inter_matrix[64];
    uint8_t scantable[64];
    uint8_t pad[8];
} MpvqState;
typedef struct MpvqRecord { uint8_t qscale, intra, dc_scale, chroma; uint32_t lambda2; } MpvqRecord;

/* vlc: intra len, intra last, inter len, inter last (NULL: plain quantiser only).  blocks[i]: the spatial samples in, the levels out.
 * overflow[i] = the quantiser's overflow flag; coded_score[i]: in = what s->coded_score[n] holds before, out = after.  nr_offset /
 * nr_sum / nr_count: s->dct_offset, s->dct_error_sum, s->dct_count (NULL nr_sum = noise reduction off); the sums are added to. */
EXPORT int ref_mpvq_batch(const MpvqState *st, const uint8_t *const *vlc, int trellis, int post, const MpvqRecord *recs, size_t n,
                          int16_t *blocks, int32_t *last_index, int32_t *overflow, int32_t *coded_score,
                          const uint16_t *nr_offset, int32_t *nr_sum, int32_t *nr_count)
{
    if (st->fdct != 0 && st->fdct != 2) return -1;
    if (trellis && !vlc) return -1;
    AVCodecContext *avctx = calloc(1, sizeof(*avctx));
    MpegEncContext *s = av_mallocz(sizeof(*s));
    int16_t (*blk)[64] = av_mallocz(12 * 64 * sizeof(int16_t));
    if (!avctx || !s || !blk) return -1;
    av_set_cpu_flags_mask(0);                                    /* portable C only, like libavref.so */
    avctx->dct_algo = st->fdct == 2 ? FF_DCT_FASTINT : FF_DCT_AUTO;
    avctx->bits_per_raw_sample = 8;
    avctx->mb_decision = FF_MB_DECISION_BITS;                    /* (clip_coeffs logs only under FF_MB_DECISION_SIMPLE) */
    s->avctx = avctx;
    ff_fdctdsp_init(&s->fdsp, avctx);
    s->idsp.perm_type = FF_IDCT_PERM_NONE;
    for (int i = 0; i < 64; i++) s->idsp.idct_permutation[i] = i;
    s->intra_scantable.scantable = st->scantable;
    memcpy(s->intra_scantable.permutated, st->scantable, 64);
    s->out_format = st->out_format; s->mpeg_quant = st->mpeg_quant; s->h263_aic = st->h263_aic;
    s->intra_quant_bias = st->intra_quant_bias; s->inter_quant_bias = st->inter_quant_bias; s->ac_esc_length = st->ac_esc_length;
    s->min_qcoeff = st->min_qcoeff; s->max_qcoeff = st->max_qcoeff;
    s->luma_elim_threshold = st->luma_elim_threshold; s->chroma_elim_threshold = st->chroma_elim_threshold;
    s->q_intra_matrix = (int (*)[64])st->q_intra_matrix;
    s->q_inter_matrix = (int (*)[64])st->q_inter_matrix;
    memcpy(s->intra_matrix, st->intra_matrix, sizeof(s->intra_matrix));
    memcpy(s->inter_matrix, st->inter_matrix, sizeof(s->inter_matrix));
    if (vlc) {
        s->intra_ac_vlc_length = (uint8_t *)vlc[0]; s->intra_ac_vlc_last_length = (uint8_t *)vlc[1];
        s->inter_ac_vlc_length = (uint8_t *)vlc[2]; s->inter_ac_vlc_last_length = (uint8_t *)vlc[3];
    }
    if (nr_sum) {
        s->dct_error_sum = (int (*)[64])nr_sum;
        s->dct_offset = (uint16_t (*)[64])nr_offset;
        s->dct_count[0] = nr_count[0]; s->dct_count[1] = nr_count[1];
    }
    s->denoise_dct = denoise_dct_c;
    s->dct_quantize = trellis ? dct_quantize_trellis_c : ff_dct_quantize_c;
    s->block = blk;

    for (size_t i = 0; i < n; i++) {
        const MpvqRecord *r = &recs[i];
        const int bn = r->chroma ? 4 : 0;
        int ovf = 0, last;
        s->mb_intra = r->intra;
        s->y_dc_scale = s->c_dc_scale = r->dc_scale;
        s->lambda2 = r->lambda2;
        s->coded_score[bn] = coded_score[i];
        memcpy(blk[bn], blocks + 64 * i, 128);
        last = s->dct_quantize(s, blk[bn], bn, r->qscale, &ovf);
        if (post) {
            if (ovf) clip_coeffs(s, blk[bn], last);
            s->block_last_index[bn] = last;
            if (s->luma_elim_threshold && !s->mb_intra && bn < 4) dct_single_coeff_elimination(s, bn, s->luma_elim_threshold);
            if (s->chroma_elim_threshold && !s->mb_intra && bn >= 4) dct_single_coeff_elimination(s, bn, s->chroma_elim_threshold);
            last = s->block_last_index[bn];
        }
        memcpy(blocks + 64 * i, blk[bn], 128);
        last_index[i] = last;
        overflow[i] = ovf;
        coded_score[i] = s->coded_score[bn];
    }
    if (nr_sum) { nr_count[0] = s->dct_count[0]; nr_count[1] = s->dct_count[1]; }
    av_free(blk); av_free(s); free(avctx);
    return 0;
}

/* the reference's ff_inv_aanscales (aandcttab.c), which the product derives from its definition */
EXPORT void ref_mpvq_inv_aanscales(uint16_t *out) { memcpy(out, ff_inv_aanscales, 64 * sizeof(uint16_t)); }

/* the functions ref_mpvq_batch installs: a test checks that they are this unit's own copies of the static quantisers */
EXPORT void ref_mpvq_impl(void **trellis, void **plain, void **denoise)
{
    *trellis = (void *)dct_quantize_trellis_c;
    *plain = (void *)ff_dct_quantize_c;
    *denoise = (void *)denoise_dct_c;
}
