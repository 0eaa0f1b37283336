/*
 * include/avdsp_b200_tables.h -- the reference's DSP function-pointer tables, restated so that
 * libavdsp_b200.so can fill them (ff_*_init_cuda) without including libav's private headers.
 *
 * Field order, types and slot signatures are the contract (they must be LAYOUT-IDENTICAL to the cited
 * reference structs, tests/test_abi_cpu.py checks sizes/offsets against oracle/_ref when it is built).
 * Nothing here is executable.
 */
#ifndef AVDSP_B200_TABLES_H
#define AVDSP_B200_TABLES_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#define AVB_RESTRICT __restrict__
#else
#define AVB_RESTRICT restrict
#endif

/* ---- libavcodec/idctdsp.h:36-43 (enum), :53-98 (struct) ---- */
enum idct_permutation_type {
    FF_IDCT_PERM_NONE, FF_IDCT_PERM_LIBMPEG2, FF_IDCT_PERM_SIMPLE,
    FF_IDCT_PERM_TRANSPOSE, FF_IDCT_PERM_PARTTRANS, FF_IDCT_PERM_SSE2,
};
typedef struct IDCTDSPContext {
    void (*put_pixels_clamped)(const int16_t *block, uint8_t *AVB_RESTRICT pixels, ptrdiff_t line_size);
    void (*put_signed_pixels_clamped)(const int16_t *block, uint8_t *AVB_RESTRICT pixels, ptrdiff_t line_size);
    void (*add_pixels_clamped)(const int16_t *block, uint8_t *AVB_RESTRICT pixels, ptrdiff_t line_size);
    void (*idct)(int16_t *block);
    void (*idct_put)(uint8_t *dest, ptrdiff_t line_size, int16_t *block);
    void (*idct_add)(uint8_t *dest, ptrdiff_t line_size, int16_t *block);
    uint8_t idct_permutation[64];
    enum idct_permutation_type perm_type;
} IDCTDSPContext;
/* idct_algo values the hook understands (libavcodec/avcodec.h FF_IDCT_*) */
#define AVB_FF_IDCT_AUTO   0
#define AVB_FF_IDCT_SIMPLE 2
#define AVB_FF_IDCT_XVID   14
#define AVB_FF_IDCT_FAAN   20

/* ---- libavcodec/proresdsp.h:31-35 ---- */
typedef struct ProresDSPContext {
    int idct_permutation_type;
    uint8_t idct_permutation[64];
    void (*idct_put)(uint16_t *out, ptrdiff_t linesize, int16_t *block, const int16_t *qmat);
} ProresDSPContext;

/* ---- libavcodec/fdctdsp.h:26-29 ---- */
typedef struct FDCTDSPContext {
    void (*fdct)(int16_t *block);
    void (*fdct248)(int16_t *block);
} FDCTDSPContext;
#define AVB_FF_DCT_AUTO    0
#define AVB_FF_DCT_FASTINT 1
#define AVB_FF_DCT_INT     2
#define AVB_FF_DCT_FAAN    6

/* ---- libavcodec/blockdsp.h:29-37 ---- */
typedef void (*op_fill_func)(uint8_t *block, uint8_t value, ptrdiff_t line_size, int h);
typedef struct BlockDSPContext {
    void (*clear_block)(int16_t *block);
    void (*clear_blocks)(int16_t *blocks);
    op_fill_func fill_block_tab[2];
} BlockDSPContext;

/* ---- libavcodec/me_cmp.h:34-63 ---- */
struct MpegEncContext;
typedef int (*me_cmp_func)(struct MpegEncContext *c, uint8_t *blk1, uint8_t *blk2, ptrdiff_t stride, int h);
typedef struct MECmpContext {
    int (*sum_abs_dctelem)(int16_t *block);
    me_cmp_func sad[6];
    me_cmp_func sse[6];
    me_cmp_func hadamard8_diff[6];
    me_cmp_func dct_sad[6];
    me_cmp_func quant_psnr[6];
    me_cmp_func bit[6];
    me_cmp_func rd[6];
    me_cmp_func vsad[6];
    me_cmp_func vsse[6];
    me_cmp_func nsse[6];
    me_cmp_func dct_max[6];
    me_cmp_func dct264_sad[6];
    me_cmp_func me_pre_cmp[6];
    me_cmp_func me_cmp[6];
    me_cmp_func me_sub_cmp[6];
    me_cmp_func mb_cmp[6];
    me_cmp_func ildct_cmp[6];
    me_cmp_func frame_skip_cmp[6];
    me_cmp_func pix_abs[2][4];
} MECmpContext;

/* ---- libavcodec/h264dsp.h:32-117 ---- */
typedef void (*h264_weight_func)(uint8_t *block, int stride, int height, int log2_denom, int weight, int offset);
typedef void (*h264_biweight_func)(uint8_t *dst, uint8_t *src, int stride, int height, int log2_denom,
                                   int weightd, int weights, int offset);
typedef struct H264DSPContext {
    h264_weight_func   weight_h264_pixels_tab[4];
    h264_biweight_func biweight_h264_pixels_tab[4];
    void (*h264_v_loop_filter_luma)(uint8_t *pix, int stride, int alpha, int beta, int8_t *tc0);
    void (*h264_h_loop_filter_luma)(uint8_t *pix, int stride, int alpha, int beta, int8_t *tc0);
    void (*h264_h_loop_filter_luma_mbaff)(uint8_t *pix, int stride, int alpha, int beta, int8_t *tc0);
    void (*h264_v_loop_filter_luma_intra)(uint8_t *pix, int stride, int alpha, int beta);
    void (*h264_h_loop_filter_luma_intra)(uint8_t *pix, int stride, int alpha, int beta);
    void (*h264_h_loop_filter_luma_mbaff_intra)(uint8_t *pix, int stride, int alpha, int beta);
    void (*h264_v_loop_filter_chroma)(uint8_t *pix, int stride, int alpha, int beta, int8_t *tc0);
    void (*h264_h_loop_filter_chroma)(uint8_t *pix, int stride, int alpha, int beta, int8_t *tc0);
    void (*h264_h_loop_filter_chroma_mbaff)(uint8_t *pix, int stride, int alpha, int beta, int8_t *tc0);
    void (*h264_v_loop_filter_chroma_intra)(uint8_t *pix, int stride, int alpha, int beta);
    void (*h264_h_loop_filter_chroma_intra)(uint8_t *pix, int stride, int alpha, int beta);
    void (*h264_h_loop_filter_chroma_mbaff_intra)(uint8_t *pix, int stride, int alpha, int beta);
    void (*h264_loop_filter_strength)(int16_t bS[2][4][4], uint8_t nnz[40], int8_t ref[2][40],
                                      int16_t mv[2][40][2], int bidir, int edges, int step,
                                      int mask_mv0, int mask_mv1, int field);
    void (*h264_idct_add)(uint8_t *dst, int16_t *block, int stride);
    void (*h264_idct8_add)(uint8_t *dst, int16_t *block, int stride);
    void (*h264_idct_dc_add)(uint8_t *dst, int16_t *block, int stride);
    void (*h264_idct8_dc_add)(uint8_t *dst, int16_t *block, int stride);
    void (*h264_idct_add16)(uint8_t *dst, const int *blockoffset, int16_t *block, int stride, const uint8_t nnzc[15 * 8]);
    void (*h264_idct8_add4)(uint8_t *dst, const int *blockoffset, int16_t *block, int stride, const uint8_t nnzc[15 * 8]);
    void (*h264_idct_add8)(uint8_t **dst, const int *blockoffset, int16_t *block, int stride, const uint8_t nnzc[15 * 8]);
    void (*h264_idct_add16intra)(uint8_t *dst, const int *blockoffset, int16_t *block, int stride, const uint8_t nnzc[15 * 8]);
    void (*h264_luma_dc_dequant_idct)(int16_t *output, int16_t *input, int qmul);
    void (*h264_chroma_dc_dequant_idct)(int16_t *block, int qmul);
    void (*h264_add_pixels8_clear)(uint8_t *dst, int16_t *block, int stride);
    void (*h264_add_pixels4_clear)(uint8_t *dst, int16_t *block, int stride);
    int (*startcode_find_candidate)(const uint8_t *buf, int size);
} H264DSPContext;

/* ---- libavcodec/qpeldsp.h (qpel_mc_func), libavcodec/h264qpel.h:27-30 ---- */
typedef void (*qpel_mc_func)(uint8_t *dst, const uint8_t *src, ptrdiff_t stride);
typedef struct H264QpelContext {
    qpel_mc_func put_h264_qpel_pixels_tab[4][16];
    qpel_mc_func avg_h264_qpel_pixels_tab[4][16];
} H264QpelContext;

/* ---- libavcodec/qpeldsp.h:69-73 (qpel_mc_func as above) ---- */
typedef struct QpelDSPContext {
    qpel_mc_func put_qpel_pixels_tab[2][16];
    qpel_mc_func avg_qpel_pixels_tab[2][16];
    qpel_mc_func put_no_rnd_qpel_pixels_tab[2][16];
} QpelDSPContext;

/* ---- libavcodec/h263dsp.h:26-29 ---- */
typedef struct H263DSPContext {
    void (*h263_h_loop_filter)(uint8_t *src, int stride, int qscale);
    void (*h263_v_loop_filter)(uint8_t *src, int stride, int qscale);
} H263DSPContext;

/* ---- libavcodec/mpegvideodsp.h:27-41 ---- */
typedef struct MpegVideoDSPContext {
    void (*gmc1)(uint8_t *dst, uint8_t *src, int srcStride, int h, int x16, int y16, int rounder);
    void (*gmc)(uint8_t *dst, uint8_t *src, int stride, int h, int ox, int oy, int dxx, int dxy, int dyx, int dyy, int shift, int r,
                int width, int height);
} MpegVideoDSPContext;

/* ---- libavcodec/h264chroma.h:25-30 ---- */
typedef void (*h264_chroma_mc_func)(uint8_t *dst, uint8_t *src, ptrdiff_t srcStride, int h, int x, int y);
typedef struct H264ChromaContext {
    h264_chroma_mc_func put_h264_chroma_pixels_tab[3];
    h264_chroma_mc_func avg_h264_chroma_pixels_tab[3];
} H264ChromaContext;

/* ---- libavcodec/hpeldsp.h:38-93 ---- */
typedef void (*op_pixels_func)(uint8_t *block, const uint8_t *pixels, ptrdiff_t line_size, int h);
typedef struct HpelDSPContext {
    op_pixels_func put_pixels_tab[4][4];
    op_pixels_func avg_pixels_tab[4][4];
    op_pixels_func put_no_rnd_pixels_tab[4][4];
    op_pixels_func avg_no_rnd_pixels_tab[4];
} HpelDSPContext;

/* ---- libavcodec/pixblockdsp.h:27-35 ---- */
typedef struct PixblockDSPContext {
    void (*get_pixels)(int16_t *AVB_RESTRICT block, const uint8_t *pixels, ptrdiff_t stride);
    void (*diff_pixels)(int16_t *AVB_RESTRICT block, const uint8_t *s1, const uint8_t *s2, ptrdiff_t stride);
} PixblockDSPContext;

/* ---- libavcodec/h264pred.h:91-110 ---- */
typedef struct H264PredContext {
    void (*pred4x4[9 + 3 + 3])(uint8_t *src, const uint8_t *topright, ptrdiff_t stride);
    void (*pred8x8l[9 + 3])(uint8_t *src, int topleft, int topright, ptrdiff_t stride);
    void (*pred8x8[4 + 3 + 4])(uint8_t *src, ptrdiff_t stride);
    void (*pred16x16[4 + 3 + 2])(uint8_t *src, ptrdiff_t stride);
    void (*pred4x4_add[2])(uint8_t *pix, int16_t *block, ptrdiff_t stride);
    void (*pred8x8l_add[2])(uint8_t *pix, int16_t *block, ptrdiff_t stride);
    void (*pred8x8l_filter_add[2])(uint8_t *pix, int16_t *block, int topleft, int topright, ptrdiff_t stride);
    void (*pred8x8_add[3])(uint8_t *pix, const int *block_offset, int16_t *block, ptrdiff_t stride);
    void (*pred16x16_add[3])(uint8_t *pix, const int *block_offset, int16_t *block, ptrdiff_t stride);
} H264PredContext;
#define AVB_AV_CODEC_ID_H264 27

/* ---- libavcodec/fft.h:36-99 (float build: FFTSample = FFTDouble = float), libavcodec/avfft.h FFTComplex ---- */
typedef float FFTSample;
typedef float FFTDouble;    /* float build, libavcodec/fft.h:39 */
typedef struct FFTComplex { FFTSample re, im; } FFTComplex;
enum fft_permutation_type { FF_FFT_PERM_DEFAULT, FF_FFT_PERM_SWAP_LSBS, FF_FFT_PERM_AVX };
enum mdct_permutation_type { FF_MDCT_PERM_NONE, FF_MDCT_PERM_INTERLEAVE };
typedef struct FFTContext {
    int nbits;
    int inverse;
    uint16_t *revtab;
    FFTComplex *tmp_buf;
    int mdct_size;
    int mdct_bits;
    FFTSample *tcos;
    FFTSample *tsin;
    void (*fft_permute)(struct FFTContext *s, FFTComplex *z);
    void (*fft_calc)(struct FFTContext *s, FFTComplex *z);
    void (*imdct_calc)(struct FFTContext *s, FFTSample *output, const FFTSample *input);
    void (*imdct_half)(struct FFTContext *s, FFTSample *output, const FFTSample *input);
    void (*mdct_calc)(struct FFTContext *s, FFTSample *output, const FFTSample *input);
    void (*mdct_calcw)(struct FFTContext *s, FFTDouble *output, const FFTSample *input);
    enum fft_permutation_type fft_permutation;
    enum mdct_permutation_type mdct_permutation;
} FFTContext;

#ifdef __cplusplus
}
#endif
#endif /* AVDSP_B200_TABLES_H */
