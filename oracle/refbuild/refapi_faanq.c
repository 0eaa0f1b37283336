/*
 * oracle/refbuild/refapi_faanq.c -- TEST INFRASTRUCTURE, NOT PRODUCT.
 *
 * The reference's encoder quantisers behind the FAAN forward DCT (FF_DCT_FAAN: s->fdsp.fdct = ff_faandct, fdctdsp.c:35-39).
 * refapi_mpvq.c is compiled once more with ff_fdctdsp_init renamed to the function below, which runs the real ff_fdctdsp_init and then
 * installs the FAAN pair, as ff_fdctdsp_init itself does for dct_algo FF_DCT_FAAN.  Everything else -- the unmodified mpegvideo_enc.c
 * with its static quantisers, the per-record loop -- is refapi_mpvq.c's.  ref_faanq_batch takes FFMpvQuantState with fdct 6.
 */
#define ff_fdctdsp_init faanq_fdctdsp_init
#define ref_mpvq_batch faanq_mpvq_batch
#define ref_mpvq_inv_aanscales faanq_mpvq_inv_aanscales
#define ref_mpvq_impl faanq_mpvq_impl
#include "refapi_mpvq.c"
#undef ff_fdctdsp_init
#include "libavcodec/faandct.h"

void ff_fdctdsp_init(FDCTDSPContext *c, AVCodecContext *avctx);

void faanq_fdctdsp_init(FDCTDSPContext *c, AVCodecContext *avctx)
{
    ff_fdctdsp_init(c, avctx);
    c->fdct = ff_faandct;
    c->fdct248 = ff_faandct248;
}

/* ref_mpvq_batch with s->fdsp.fdct = ff_faandct; the state's fdct must be 6 */
EXPORT int ref_faanq_batch(const MpvqState *st, const uint8_t *const *vlc, int trellis, int post, const MpvqRecord *recs, size_t n,
                           int16_t *blocks, int32_t *last_index, int32_t *overflow, int32_t *coded_score,
                           const uint16_t *nr_offset, int32_t *nr_sum, int32_t *nr_count)
{
    if (st->fdct != 6) return -1;
    MpvqState s = *st;
    s.fdct = 0;                                                  /* (refapi_mpvq.c's own check; the transform comes from the init above) */
    return faanq_mpvq_batch(&s, vlc, trellis, post, recs, n, blocks, last_index, overflow, coded_score, nr_offset, nr_sum, nr_count);
}
