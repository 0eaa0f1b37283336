/*
 * oracle/oracle_api.h -- TEST INFRASTRUCTURE, NOT PRODUCT.
 *
 * One flat C API, implemented twice:
 *   orc_*  oracle/port/*.c          plain-C restatement of the reference algorithms
 *   ref_*  oracle/refbuild/refapi.c thin calls into the UNMODIFIED reference, compiled
 *                                   from /root/reference into oracle/_ref/libavref.so
 * tests/ drive both with the same ctypes prototypes, so every restated function is
 * byte-compared with the real reference in this container; the port (and the prebuilt
 * _ref .so) then travel to the GPU box as the checker for the CUDA path.
 *
 * Only tests/, __graft_entry__.smoke() and bench.py's CPU legs may use this API.
 */
#ifndef ORACLE_API_H
#define ORACLE_API_H
#include <stdint.h>
#include <stddef.h>

#ifndef ORC_PREFIX
#define ORC_PREFIX orc_
#endif
#define ORC_CAT2(a, b) a##b
#define ORC_CAT(a, b) ORC_CAT2(a, b)
#define ORC(n) ORC_CAT(ORC_PREFIX, n)

#ifdef __cplusplus
extern "C" {
#endif

/* ---- IDCTDSPContext / BlockDSPContext (libavcodec/idctdsp.h:53-98, blockdsp.h:32-37) */
void ORC(simple_idct_put)(uint8_t *dst, ptrdiff_t stride, int16_t *block);
void ORC(simple_idct_add)(uint8_t *dst, ptrdiff_t stride, int16_t *block);
void ORC(simple_idct)(int16_t *block);
void ORC(put_pixels_clamped)(const int16_t *block, uint8_t *pixels, ptrdiff_t stride);
void ORC(put_signed_pixels_clamped)(const int16_t *block, uint8_t *pixels, ptrdiff_t stride);
void ORC(add_pixels_clamped)(const int16_t *block, uint8_t *pixels, ptrdiff_t stride);
void ORC(clear_block)(int16_t *block);
void ORC(clear_blocks)(int16_t *blocks);
void ORC(fill_block)(int w16, uint8_t *block, uint8_t value, ptrdiff_t stride, int h);

/* the 10-bit instance (ff_simple_idct_put_10 / _add_10 / _10, simple_idct_template.c BIT_DEPTH == 10: 16-bit samples, `stride` in bytes),
 * what ff_idctdsp_init installs for bits_per_raw_sample == 10 (idctdsp.c:151-155).  mode 0 put, 1 add, 2 in place (dst ignored) */
void ORC(simple_idct10)(int mode, uint8_t *dst, ptrdiff_t stride, int16_t *block);

/* batch driver used for parity at scale and for CPU timing: block i -> frame + dst_off[i].
 * mode 0 = idct_put, 1 = idct_add, 2 = idct (in place, frame ignored).
 * nthreads > 1 splits the block range over pthreads. The blocks array is clobbered exactly
 * as the per-block functions clobber it. */
void ORC(idct_batch)(int mode, int16_t *blocks, uint8_t *frame, const uint32_t *dst_off,
                     ptrdiff_t stride, size_t n, int nthreads);

/* ---- FDCTDSPContext (libavcodec/fdctdsp.h:26-29): 0 = jpeg_fdct_islow_8, 1 = fdct248_islow_8,
 *      2 = fdct_ifast, 3 = fdct_ifast248, 4 = jpeg_fdct_islow_10, 5 = fdct248_islow_10 (bits_per_raw_sample == 10, fdctdsp.c:31-33) */
void ORC(fdct)(int which, int16_t *block);

/* ---- H264DSPContext (libavcodec/h264dsp.h:41-117), 8-bit ---- */
/* which: 0 idct_add, 1 idct8_add, 2 idct_dc_add, 3 idct8_dc_add */
void ORC(h264_idct)(int which, uint8_t *dst, int16_t *block, int stride);
/* which: 0 idct_add16, 1 idct_add16intra, 2 idct8_add4, 3 idct_add8 (dst2 = {cb, cr}), 4 idct_add8_422 (the table entry for
 * chroma_format_idc 2, h264dsp.c:81-84) */
void ORC(h264_idct_mb)(int which, uint8_t *dst, uint8_t **dst2, const int *block_offset,
                       int16_t *block, int stride, const uint8_t *nnzc);
void ORC(h264_luma_dc_dequant_idct)(int16_t *output, int16_t *input, int qmul);
void ORC(h264_chroma_dc_dequant_idct)(int16_t *block, int qmul);
void ORC(h264_chroma422_dc_dequant_idct)(int16_t *block, int qmul);   /* the chroma_format_idc 2 entry, h264dsp.c:87-90 */
/* which: 0 v_luma 1 h_luma 2 v_luma_intra 3 h_luma_intra 4 v_chroma 5 h_chroma
 *        6 v_chroma_intra 7 h_chroma_intra ; tc0 ignored for intra
 *        8 h_luma_mbaff 9 h_luma_mbaff_intra 10 h_chroma_mbaff 11 h_chroma_mbaff_intra, and the chroma_format_idc 2 entries
 *        12 h_chroma422 13 h_chroma422_intra 14 h_chroma422_mbaff 15 h_chroma422_mbaff_intra (h264dsp.c:104-122) */
void ORC(h264_loop_filter)(int which, uint8_t *pix, int stride, int alpha, int beta,
                           const int8_t *tc0);

/* QpelDSPContext (libavcodec/qpeldsp.h:69-73, qpeldsp.c:39-766): MPEG-4 quarter-pel motion compensation.
 * kind 0 put_qpel_pixels_tab, 1 put_no_rnd_qpel_pixels_tab, 2 avg_qpel_pixels_tab; sidx 0 = 16x16, 1 = 8x8;
 * mc = x + 4 * y quarter-pel phase.  dst and src share `stride`; reads rows 0..N and columns 0..N of src. */
void ORC(mpeg4_qpel)(int kind, int sidx, int mc, uint8_t *dst, const uint8_t *src, ptrdiff_t stride);

/* PixblockDSPContext (libavcodec/pixblockdsp.h:27-35, pixblockdsp_template.c): kind 0 get_pixels (s2 unused),
 * kind 1 diff_pixels = s1 - s2; 8x8 samples -> int16 block, row-major */
void ORC(pixblock)(int kind, int16_t *block, const uint8_t *s1, const uint8_t *s2, ptrdiff_t stride);

/* H.264 intra prediction, H264PredContext for codec H.264, 8 bit, 4:2:0 (libavcodec/h264pred.h:91-110,
 * h264pred_template.c): the block at `src` is overwritten from its neighbours in the same plane.
 *   tab 0 pred4x4[mode 0..11]  (topright -> 4 samples, only read by DIAG_DOWN_LEFT / VERT_LEFT)
 *       1 pred8x8l[mode 0..11] (has_topleft / has_topright as the decoder passes them)
 *       2 pred8x8[mode 0..10]  (chroma: DC, HOR, VERT, PLANE, LEFT_DC, TOP_DC, DC_128, 4 x "ALZHEIMER" DC)
 *       3 pred16x16[mode 0..6] (DC, HOR, VERT, PLANE, LEFT_DC, TOP_DC, DC_128) */
void ORC(h264_pred)(int tab, int mode, uint8_t *src, const uint8_t *topright, int has_topleft, int has_topright, ptrdiff_t stride);
/* lossless (transform-bypass) vertical / horizontal prediction + residual: tab 0 pred4x4_add  1 pred8x8l_add
 * 2 pred8x8l_filter_add  3 pred8x8_add (4 blocks at block_offset[0..3])  4 pred16x16_add (16 blocks);
 * mode 0 vertical, 1 horizontal; the consumed coefficients are zeroed. */
void ORC(h264_pred_add)(int tab, int mode, uint8_t *pix, const int *block_offset, int16_t *block, int has_topleft,
                        int has_topright, ptrdiff_t stride);

/* MPEG-1/2/4 and H.263 inverse quantisation of one 8x8 block in place: MpegEncContext.dct_unquantize_*
 * (libavcodec/mpegvideo.c:51-270), simple-IDCT permutation (none).
 *   kind 0 mpeg1_intra  1 mpeg1_inter  2 mpeg2_intra  3 mpeg2_intra_bitexact (with mismatch control)  4 mpeg2_inter
 *        5 h263_intra   6 h263_inter
 *   n = block number inside the macroblock (< 4: y_dc_scale, else c_dc_scale), last_index = block_last_index[n]. */
void ORC(mpeg_dequant)(int kind, int16_t *block, int n, int qscale, int last_index, int y_dc_scale, int c_dc_scale,
                       const uint16_t *intra_matrix, const uint16_t *inter_matrix, int alternate_scan, int h263_aic, int ac_pred);
/* ScanTable.permutated of intra_scantable and ScanTable.raster_end of inter_scantable (idctdsp.c:28-47,
 * mpegvideo.c:299-317) for the zigzag (0) or alternate vertical (1) scan */
void ORC(mpeg_scantables)(int alternate_scan, uint8_t *permutated, uint8_t *raster_end);

/* ---- MECmpContext.quant_psnr / bit / rd (libavcodec/me_cmp.c:621-782): the three comparison functions that run the encoder's own
 * quantiser (s->fast_dct_quantize = ff_dct_quantize_c, libavcodec/mpegvideo_enc.c:4371-4450), count VLC bits from the codec's
 * length tables and / or reconstruct through s->dct_unquantize_* and the simple IDCT.  OrcEncState = the MpegEncContext fields they read.
 *   kind 14 quant_psnr, 15 bit, 16 rd; sidx 0 = the 16-wide wrappers (h 16 or 8), 1 = 8x8 (h 8)
 *   side[0] = s->block_last_index[0] after the call, side[1] = s->mb_intra after the call (quant_psnr clears it) */
typedef struct OrcEncState {
    int32_t fdct_sel;        /* s->fdsp.fdct: 0 ff_jpeg_fdct_islow_8 (FF_DCT_AUTO), 2 ff_fdct_ifast (FF_DCT_FASTINT) */
    int32_t dequant;         /* s->dct_unquantize_intra / _inter (mpegvideo_enc.c:1613-1622): 0 mpeg1, 1 mpeg2, 2 mpeg2 with AV_CODEC_FLAG_BITEXACT, 3 h263 */
    int32_t qscale, mb_intra, y_dc_scale, c_dc_scale, h263_aic, ac_pred, alternate_scan;
    int32_t intra_quant_bias, inter_quant_bias, ac_esc_length;
    uint16_t intra_matrix[64], inter_matrix[64];
    const uint8_t *intra_ac_vlc_length, *intra_ac_vlc_last_length, *inter_ac_vlc_length, *inter_ac_vlc_last_length;   /* [64 * 128], UNI_AC_ENC_INDEX */
    const uint8_t *luma_dc_vlc_length;                                                                               /* [512] */
} OrcEncState;
int ORC(me_cmp_quant)(int kind, int sidx, const OrcEncState *st, uint8_t *b1, uint8_t *b2, ptrdiff_t stride, int h, int32_t *side);
/* s->q_intra_matrix[qscale] / s->q_inter_matrix[qscale] as ff_convert_matrix() builds them (mpegvideo_enc.c:84-160), and
 * s->intra_scantable.scantable (the order the quantiser walks) */
void ORC(enc_qmatrices)(const OrcEncState *st, int32_t *q_intra, int32_t *q_inter, uint8_t *scantable);

/* Deblocking DECISIONS for one progressive 4:2:0 8-bit picture (SURVEY 8f rank 1; h264_deblock_params_hbd: of bit_depth 8, 9 or 10): what loop_filter() ->
 * fill_filter_caches() -> ff_h264_filter_mb() (libavcodec/h264_slice.c:2198-2262, :1972-2196,
 * libavcodec/h264_loopfilter.c:420-846) decide per macroblock -- which edges are filtered with which
 * (alpha, beta, tc0 | bS 4).  Inputs are the decoder's own side-information arrays in the decoder's layouts:
 *   mb_type, qscale, cbp, slice_table : [mb_h * mb_stride], mb_stride = mb_w + 1, index mb_x + mb_y * mb_stride
 *                                       (the extra column is padding and is never read here)
 *   nnz        : [mb_h * mb_stride][48]   H264Context.non_zero_count (luma 4x4 block k at [k], raster inside the MB)
 *   mv0 / mv1  : [4 * mb_h][4 * mb_w][2]  H264Picture.motion_val[list], b_stride = 4 * mb_w, quarter-pel
 *   ref0 / ref1: [mb_h * mb_stride][4]    H264Picture.ref_index[list] per 8x8
 *   slice_params: per slice_num 133 int32 = { slice_alpha_c0_offset, slice_beta_offset, deblocking_filter,
 *                 list_count, qp_thresh, ref2frm[2][64] }  (H264SliceContext / H264Context.ref2frm, h264dec.h:186,538)
 *   chroma_qp_table: PPS.chroma_qp_table[2][64] (h264_ps.h:124)
 * At 9 / 10 bit qscale and chroma_qp_table are in the decoder's QP' scale (0..51 + 6 * (bit_depth - 8)), and qp_thresh carries its
 * + 6 * (bit_depth - 8) term (h264_slice.c:1815-1820); the records keep the 8-bit-scale alpha / beta / tc0 the filters are called with.
 * out: mb_w * mb_h records of 104 bytes, raster order, in the layout of FFH264DeblockMB (include/avdsp_b200.h):
 *   alpha[2][4] beta[2][4] tc0[2][4][4] intra[2] calpha[2][2][2] cbeta[2][2][2] ctc0[2][2][2][4] cintra[2][2] pad[2];
 *   an edge that is not filtered has alpha = beta = 0. Returns 0, or -1 for n_slices > 32 or a bit_depth other than 8 / 9 / 10. */
int ORC(h264_deblock_params)(int mb_w, int mb_h, const uint32_t *mb_type, const int8_t *qscale, const uint8_t *nnz,
                             const uint16_t *cbp, const uint16_t *slice_table, const int16_t *mv0, const int16_t *mv1,
                             const int8_t *ref0, const int8_t *ref1, const int32_t *slice_params, int n_slices,
                             const uint8_t *chroma_qp_table, int cabac, int transform_8x8_mode, uint8_t *out);
int ORC(h264_deblock_params_hbd)(int bit_depth, int mb_w, int mb_h, const uint32_t *mb_type, const int8_t *qscale, const uint8_t *nnz,
                                 const uint16_t *cbp, const uint16_t *slice_table, const int16_t *mv0, const int16_t *mv1,
                                 const int8_t *ref0, const int8_t *ref1, const int32_t *slice_params, int n_slices,
                                 const uint8_t *chroma_qp_table, int cabac, int transform_8x8_mode, uint8_t *out);
/* the pictures of the following h264_deblock_params / h264_deblock_picture_with calls are fields (h->picture_structure != PICT_FRAME; their
 * mb_type entries must carry MB_TYPE_INTERLACED, 0x80): mvy_limit 2, bS 3 on horizontal intra macroblock edges (h264_loopfilter.c:551-557,723) */
void ORC(h264_deblock_picture_structure)(int field_picture);
/* chroma_format_idc 2 for the following h264_deblock_params calls while ext != NULL: the four horizontal chroma edges of every macroblock
 * (chroma rows 0, 4, 8, 12; h264_loopfilter.c:633,693-700) are written to ext + 52 * mb as alpha[2 planes][4], beta[2][4], tc0[2][4][4], intra[2], pad[2];
 * the 104-byte record keeps luma and the vertical chroma edges (whose tc0 entries then cover four of sixteen lines) */
void ORC(h264_deblock_chroma422)(uint8_t *ext);
/* widx: 0..3 = width 16,8,4,2 */
void ORC(h264_weight)(int widx, uint8_t *block, int stride, int height, int log2_denom,
                      int weight, int offset);
void ORC(h264_biweight)(int widx, uint8_t *dst, uint8_t *src, int stride, int height,
                        int log2_denom, int weightd, int weights, int offset);
void ORC(h264_add_pixels_clear)(int w8, uint8_t *dst, int16_t *block, int stride);

/* ---- SwsContext per-line slots (libswscale/swscale_internal.h:62-110,312-330,478-535): the functions sws_init_swscale()
 * (swscale.c:723-769) / ff_sws_init_output_funcs() (output.c:1357-1590) install in a context for a yuv420p source, the destination
 * format dst_fmt (AV_PIX_FMT_* value) and `flags`, called on caller-made lines.  The colour settings of sws_set_colorspace apply.
 *   hscale:  hyScale = hcScale = hScale8To15_c (dst int16[dstW]) or hScale8To19_c (dst int32[dstW]) when dst_fmt is 16-bit planar
 *   hfast:   hyscale_fast_c (chroma 0: dst1 / src1 only) or hcscale_fast_c (chroma 1)
 *   plane:   yuv2plane1 (filterSize 0, src[0]) / yuv2planeX of dst_fmt's depth; lines are int16, int32 for 16-bit destinations
 *   nv12:    yuv2nv12cX_c (dst_fmt nv12 / nv21), chrDither8 = 64
 *   packed:  kind 1 yuv2packed1 (lumSrc[0], chr*[0..1], uvalpha), 2 yuv2packed2 (two lines each, yalpha / uvalpha), 0 yuv2packedX
 * Returns 0, -1 when the reference would not install that slot (or the request is outside what the port restates). */
/*   range:   kind 0 lumRangeFromJpeg_c (dst1), 1 chrRangeFromJpeg_c (dst1, dst2), 2 lumRangeToJpeg_c, 3 chrRangeToJpeg_c: c->lumConvertRange /
 *            c->chrConvertRange of a yuvj420p -> yuv420p (0, 1) or yuv420p -> yuvj420p (2, 3) context (swscale.c:166-197,748-757) */
/* SwsFilter vectors for the sws_* calls that follow (libswscale/swscale.h:106-117): which 0 lumH, 1 lumV, 2 chrH, 3 chrV; side 0 srcFilter,
 * 1 dstFilter; length 0 clears.  The coefficient array must stay alive while it is set. */
void ORC(sws_set_filter)(int which, int side, const double *coeff, int length);
int ORC(sws_line_range)(int kind, int16_t *dst1, int16_t *dst2, int width);
int ORC(sws_line_hscale)(int dst_fmt, int flags, void *dst, int dstW, const uint8_t *src, const int16_t *filter, const int32_t *filterPos, int filterSize);
int ORC(sws_line_hfast)(int chroma, int16_t *dst1, int16_t *dst2, int dstW, const uint8_t *src1, const uint8_t *src2, int srcW, int xInc);
int ORC(sws_line_plane)(int dst_fmt, const int16_t *filter, int filterSize, const void *const *src, uint8_t *dest, int dstW, const uint8_t *dither, int offset);
int ORC(sws_line_nv12)(int dst_fmt, const int16_t *chrFilter, int chrFilterSize, const int16_t *const *chrU, const int16_t *const *chrV, uint8_t *dest, int chrDstW);
int ORC(sws_line_packed)(int dst_fmt, int flags, int kind, const int16_t *lumFilter, const int16_t *const *lumSrc, int lumFilterSize,
                         const int16_t *chrFilter, const int16_t *const *chrU, const int16_t *const *chrV, int chrFilterSize,
                         uint8_t *dest, int dstW, int yalpha, int uvalpha, int y);

/* ---- the 9 / 10-bit instances of H264DSPContext / H264QpelContext / H264ChromaContext (ff_h264dsp_init(c, bits, idc), ff_h264qpel_init(c, bits),
 * ff_h264chroma_init(c, bits); bit_depth_template.c:49-67: uint16 samples, int32 coefficients).  `which` / `widx` / `sidx` / `mc` number the
 * entries like the 8-bit functions above; strides are in BYTES; dc_dequant kind 0 luma (out, in), 1 chroma 4:2:0, 2 chroma 4:2:2 (in place in `out`) */
void ORC(h264_hbd_idct)(int bits, int which, uint8_t *dst, int32_t *block, int stride);
void ORC(h264_hbd_idct_mb)(int bits, int which, uint8_t *dst, uint8_t **dst2, const int *block_offset, int32_t *block, int stride, const uint8_t *nnzc);
void ORC(h264_hbd_dc_dequant)(int bits, int kind, int32_t *out, int32_t *in, int qmul);
void ORC(h264_hbd_add_pixels_clear)(int bits, int w8, uint8_t *dst, int32_t *block, int stride);
void ORC(h264_hbd_weight)(int bits, int widx, uint8_t *block, int stride, int height, int log2_denom, int weight, int offset);
void ORC(h264_hbd_biweight)(int bits, int widx, uint8_t *dst, uint8_t *src, int stride, int height, int log2_denom, int weightd, int weights, int offset);
void ORC(h264_hbd_loop_filter)(int bits, int which, uint8_t *pix, int stride, int alpha, int beta, const int8_t *tc0);
void ORC(h264_hbd_qpel)(int bits, int avg, int sidx, int mc, uint8_t *dst, const uint8_t *src, ptrdiff_t stride);
void ORC(h264_hbd_chroma)(int bits, int avg, int widx, uint8_t *dst, uint8_t *src, ptrdiff_t stride, int h, int x, int y);
/* H264PredContext for codec H.264, 9 / 10 bit, 4:2:0: tab / mode as h264_pred and h264_pred_add above; block_offset[] and stride in bytes */
void ORC(h264_hbd_pred)(int bits, int tab, int mode, uint8_t *src, const uint8_t *topright, int has_topleft, int has_topright, ptrdiff_t stride);
void ORC(h264_hbd_pred_add)(int bits, int tab, int mode, uint8_t *pix, const int *block_offset, int32_t *block, int has_topleft, int has_topright, ptrdiff_t stride);
/* chroma_format_idc 2: the pred8x8[] / pred8x8_add[] entries become the 8 x 16 functions (h264pred.c:477-563, h264pred_template.c:502-838,
 * 1326-1354).  bits 8 (uint8 samples, int16 residual) / 9 / 10 (uint16, int32); mode = the pred8x8[] index 0..10; add_mode 0 vertical,
 * 1 horizontal; stride and block_offset[] in bytes */
void ORC(h264_pred422)(int bits, int mode, uint8_t *src, ptrdiff_t stride);
void ORC(h264_pred422_add)(int bits, int add_mode, uint8_t *pix, const int *block_offset, void *block, ptrdiff_t stride);

/* ---- H264QpelContext / H264ChromaContext (h264qpel.h:27-30, h264chroma.h:25-30) ---- */
/* sidx 0..3 = 16,8,4,2 ; mc = (mx&3) + 4*(my&3) */
void ORC(h264_qpel)(int avg, int sidx, int mc, uint8_t *dst, const uint8_t *src, ptrdiff_t stride);
/* widx 0..2 = 8,4,2 */
void ORC(h264_chroma)(int avg, int widx, uint8_t *dst, uint8_t *src, ptrdiff_t stride, int h,
                      int x, int y);

/* ---- HpelDSPContext (hpeldsp.h:45-93) ----
 * tab 0 put, 1 avg, 2 put_no_rnd, 3 avg_no_rnd ; sidx 0..3 = 16,8,4,2 ; dxy 0..3 */
int ORC(hpel)(int tab, int sidx, int dxy, uint8_t *block, const uint8_t *pixels,
              ptrdiff_t line_size, int h);

/* ---- MECmpContext (me_cmp.h:39-63) ----
 * kind: 0 pix_abs[sidx][dxy] (sidx 0 = 16 wide, 1 = 8 wide)
 *       1 sad[sidx] 2 sse[sidx] (sidx 2 = 4 wide) 3 hadamard8_diff[sidx]
 *       4 vsad[sidx] 5 vsse[sidx] 6 nsse[sidx] (weight 8, NULL ctx)
 *       7 hadamard8 intra (me_cmp[4..5]) 8 vsad_intra 9 vsse_intra
 *      10 sum_abs_dctelem(blk1 as int16[64]) */
int ORC(me_cmp)(int kind, int sidx, int dxy, const uint8_t *blk1, const uint8_t *blk2,
                ptrdiff_t stride, int h);
/* exhaustive search restating motion_est_template.c:620-655 for config 4: for each 16x16 MB
 * of cur, search ref within +-range clipped so the block stays inside the picture, SAD16,
 * lambda 0, strict-< argmin in raster order.  out[3*mb] = mx, my, sad.  MB rows
 * [mb_y0, mb_y1). */
void ORC(full_search)(const uint8_t *cur, const uint8_t *ref, int stride, int w, int h,
                      int range, int mb_y0, int mb_y1, int32_t *out, int nthreads);

/* ---- libswscale (boundary B) ---- */
/* whole-frame yuv420p -> rgb24 through sws_getContext/sws_scale semantics
 * (swscale.h:159-207). flags are the reference's SWS_* bit values. Returns number of output
 * lines, <0 on error. */
int ORC(sws_yuv420p_to_rgb24)(const uint8_t *const src[3], const int src_stride[3], int src_w,
                              int src_h, uint8_t *dst, int dst_stride, int dst_w, int dst_h,
                              int flags);
/* whole-frame yuv420p -> yuv420p scaling (hscale + yuv2planeX vertical path) */
int ORC(sws_yuv420p_to_yuv420p)(const uint8_t *const src[3], const int src_stride[3], int src_w,
                                int src_h, uint8_t *const dst[3], const int dst_stride[3],
                                int dst_w, int dst_h, int flags);
/* filter bank as designed by initFilter (utils.c:249-632) with the geometry sws_init_context
 * (utils.c:887-1340) derives for yuv420p -> (to_rgb ? rgb24 : yuv420p).
 * which: 0 hLum, 1 hChr, 2 vLum, 3 vChr.  Fills filter (int16, n*fsize) and pos (int32, n), where
 * n = number of output samples of that axis (returned in *n_out); returns fsize (<0 on error).
 * filter_align is forced to 1 (the padding taps are zero under SWS_BITEXACT). */
/* Any source format the product takes over.  Planar 8-bit YUV of any chroma sub-sampling: src_fmt = AV_PIX_FMT_YUV420P 0, YUV422P 4,
 * YUV444P 5, YUV410P 6, YUV411P 7, YUV440P 31; packed (src[0] / ss[0] only): YUYV422 1, RGB24 2, BGR24 3, UYVY422 15
 * (libavutil/pixfmt.h).  dst_fmt 2 = rgb24, 3 = bgr24 (dst[0] only), 0 = yuv420p.  One frame through sws_getContext + sws_scale;
 * returns the lines written. */
/* colour settings for the following sws_planar calls (sws_setColorspaceDetails, utils.c:807-835): inv_table = ff_yuv2rgb_coeffs[] row,
 * src_range 1 = full-range yuv, brightness / contrast / saturation in 16.16; NULL restores sws_getContext's defaults */
void ORC(sws_set_colorspace)(const int inv_table[4], int src_range, int brightness, int contrast, int saturation);
int ORC(sws_planar)(int src_fmt, const uint8_t *const src[3], const int ss[3], int sw, int sh, int dst_fmt,
                    uint8_t *const dst[3], const int dstride[3], int dw, int dh, int flags);
/* Semi-planar sources: sws_getContext(sw, sh, AV_PIX_FMT_NV12 / NV21, dw, dh, dst_fmt, flags) + sws_scale of one frame
 * (chroma read through nv12ToUV_c / nv21ToUV_c, libswscale/input.c:475-497; same-size planar output through
 * nv12ToPlanarWrapper, swscale_unscaled.c:160-181).  dst_fmt 2 = rgb24 (dst[0] only), 0 = yuv420p.  Returns lines written. */
int ORC(sws_nv12)(int nv21, const uint8_t *y, int ystride, const uint8_t *uv, int uvstride, int sw, int sh, int dst_fmt,
                  uint8_t *const dst[3], const int dstride[3], int dw, int dh, int flags);
int ORC(sws_get_filter)(int which, int to_rgb, int src_w, int src_h, int dst_w, int dst_h, int flags,
                        int16_t *filter, int32_t *pos, int cap, int *n_out);
/* yuv->rgb 24 bpp LUTs (yuv2rgb.c:671-863) with the default colourspace (ITU601, limited range):
 * ytab[1024]; rv, gu, gv, bu int32[256]: byte offsets into ytab (gv: plain int added to gu). */
void ORC(sws_rgb24_tables)(uint8_t *ytab, int32_t *rv, int32_t *gu, int32_t *gv, int32_t *bu);

/* ---- float FFT / MDCT (fft.h:73-99) : in-place complex FFT of 2^nbits points (permute +
 *      calc), inverse != 0 for the inverse transform; imdct/mdct with scale ---- */
void ORC(fft)(int nbits, int inverse, float *z /* 2 << nbits floats */);
void ORC(imdct_half)(int nbits, double scale, float *out, const float *in);
void ORC(imdct_calc)(int nbits, double scale, float *out, const float *in);
void ORC(mdct_calc)(int nbits, double scale, float *out, const float *in);

#ifdef __cplusplus
}
#endif
#endif
