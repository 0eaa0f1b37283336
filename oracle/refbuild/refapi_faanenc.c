/*
 * oracle/refbuild/refapi_faanenc.c -- TEST INFRASTRUCTURE, NOT PRODUCT.
 *
 * The reference's quant_psnr / bit / rd comparison functions on an encoder context whose forward DCT is ff_faandct (FF_DCT_FAAN).
 * refapi_enc.c is compiled once more with ff_fdctdsp_init renamed to the function below, which runs the real ff_fdctdsp_init and then
 * installs the FAAN pair, as ff_fdctdsp_init itself does for dct_algo FF_DCT_FAAN; its two entry points are renamed ref_faanenc_*.
 * ff_convert_matrix treats ff_faandct like the islow transform (mpegvideo_enc.c:95-99), which the reused contexts get.
 */
#define ff_fdctdsp_init faanenc_fdctdsp_init
#define ref_me_cmp_quant ref_faanenc_me_cmp_quant
#define ref_enc_qmatrices ref_faanenc_qmatrices
#include "refapi_enc.c"
#undef ff_fdctdsp_init
#include "libavcodec/faandct.h"

void ff_fdctdsp_init(FDCTDSPContext *c, AVCodecContext *avctx);

void faanenc_fdctdsp_init(FDCTDSPContext *c, AVCodecContext *avctx)
{
    ff_fdctdsp_init(c, avctx);
    c->fdct = ff_faandct;
    c->fdct248 = ff_faandct248;
}
