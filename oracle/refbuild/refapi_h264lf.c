/*
 * oracle/refbuild/refapi_h264lf.c -- TEST INFRASTRUCTURE, NOT PRODUCT.
 *
 * ref_h264_deblock_params(): the reference's own deblocking DECISIONS for one picture, at bit depth 8, 9 or 10.  The decision code is the
 * unmodified libavcodec/h264_loopfilter.c (ff_h264_filter_mb_fast -> ff_h264_filter_mb, :420-437, :716-846), compiled
 * from /root/reference.  It is driven the way loop_filter() drives it (h264_slice.c:2198-2262): for each macroblock in
 * raster order fill the slice context's neighbour caches, set sl->chroma_qp[], call ff_h264_filter_mb_fast().  The
 * twelve H264DSPContext loop-filter slots are replaced by recorders, so instead of filtering pixels every call leaves
 * its (alpha, beta, tc0 | intra) in the macroblock's record -- which is exactly the input of the batched deblocking
 * kernel.  fill_filter_caches()/fill_filter_caches_inter() are static in h264_slice.c (:1972-2196) and cannot be
 * linked; gather_caches() below restates them for progressive pictures (the only part of this file with logic of its
 * own; MBAFF/field branches are left out).
 */
#define ORC_PREFIX ref_
#include "../oracle_api.h"

#include <stdlib.h>
#include <string.h>

#include "libavcodec/h264dec.h"
#include "libavcodec/h264_ps.h"
#include "libavcodec/mpegutils.h"

/* ---- recorders --------------------------------------------------------------------------------------------- */
enum { REC_LS = 64, REC_UVLS = 32 };                 /* fake picture pitches: offsets identify the edge */
static uint8_t fake_y[16 * REC_LS], fake_cb[16 * REC_UVLS], fake_cr[16 * REC_UVLS];       /* (16 chroma rows: 4:2:2) */
static uint8_t *cur_ext;                             /* 4:2:2: the 52-byte record of the horizontal chroma edges, NULL for 4:2:0 */
static uint8_t *g_ext422;
void ref_h264_deblock_chroma422(uint8_t *ext) { g_ext422 = ext; }
static uint8_t *cur_rec;                             /* 104-byte record being written (layout: oracle_api.h) */

enum { O_ALPHA = 0, O_BETA = 8, O_TC0 = 16, O_INTRA = 48, O_CALPHA = 50, O_CBETA = 58, O_CTC0 = 66, O_CINTRA = 98 };

static void rec_luma(int dir, uint8_t *pix, int alpha, int beta, const int8_t *tc0)
{
    int off = (int)(pix - fake_y), e = dir ? off / (4 * REC_LS) : off / 4;
    cur_rec[O_ALPHA + 4 * dir + e] = alpha;
    cur_rec[O_BETA + 4 * dir + e]  = beta;
    if (tc0) memcpy(cur_rec + O_TC0 + 16 * dir + 4 * e, tc0, 4);
    else     cur_rec[O_INTRA + dir] |= 1 << e;
}
static void rec_chroma(int dir, uint8_t *pix, int alpha, int beta, const int8_t *tc0)
{
    int plane = pix >= fake_cr && pix < fake_cr + sizeof(fake_cr);
    int off = (int)(pix - (plane ? fake_cr : fake_cb)), e = dir ? off / (4 * REC_UVLS) : off / 4;
    if (cur_ext && dir) {                            /* chroma_format_idc 2: rows 0, 4, 8, 12 of the 8 x 16 chroma macroblock */
        cur_ext[4 * plane + e] = alpha; cur_ext[8 + 4 * plane + e] = beta;
        if (tc0) memcpy(cur_ext + 16 + 16 * plane + 4 * e, tc0, 4);
        else     cur_ext[48 + plane] |= 1 << e;
        return;
    }
    int i = (plane * 2 + dir) * 2 + e;
    cur_rec[O_CALPHA + i] = alpha;
    cur_rec[O_CBETA + i]  = beta;
    if (tc0) memcpy(cur_rec + O_CTC0 + 4 * i, tc0, 4);
    else     cur_rec[O_CINTRA + plane * 2 + dir] |= 1 << e;
}
/* "h" filters act across vertical edges (dir 0), "v" filters across horizontal edges (dir 1) */
static void r_h_luma(uint8_t *p, int s, int a, int b, int8_t *tc)   { rec_luma(0, p, a, b, tc); }
static void r_v_luma(uint8_t *p, int s, int a, int b, int8_t *tc)   { rec_luma(1, p, a, b, tc); }
static void r_h_luma_i(uint8_t *p, int s, int a, int b)             { rec_luma(0, p, a, b, NULL); }
static void r_v_luma_i(uint8_t *p, int s, int a, int b)             { rec_luma(1, p, a, b, NULL); }
static void r_h_chroma(uint8_t *p, int s, int a, int b, int8_t *tc) { rec_chroma(0, p, a, b, tc); }
static void r_v_chroma(uint8_t *p, int s, int a, int b, int8_t *tc) { rec_chroma(1, p, a, b, tc); }
static void r_h_chroma_i(uint8_t *p, int s, int a, int b)           { rec_chroma(0, p, a, b, NULL); }
static void r_v_chroma_i(uint8_t *p, int s, int a, int b)           { rec_chroma(1, p, a, b, NULL); }

/* ---- neighbour caches (restates h264_slice.c:1972-2196 for progressive frames) ------------------------------ */
static void gather_list(const H264Context *h, H264SliceContext *sl, int mb_type, int top_xy, int left_xy,
                        int top_type, int left_type, int mb_xy, int list)
{
    const int bs = h->b_stride;
    int16_t (*mv)[2] = &sl->mv_cache[list][scan8[0]];
    int8_t *rc = &sl->ref_cache[list][scan8[0]];
    int i, r;
    if (IS_INTER(mb_type) || IS_DIRECT(mb_type)) {
        if (USES_LIST(top_type, list)) {                         /* bottom 4x4 row of the MB above */
            const int *r2f = &h->ref2frm[h->slice_table[top_xy] & (MAX_SLICES - 1)][list][2];
            const int b_xy = h->mb2b_xy[top_xy] + 3 * bs;
            memcpy(mv - 8, h->cur_pic.motion_val[list][b_xy], 16);
            rc[0 - 8] = rc[1 - 8] = r2f[h->cur_pic.ref_index[list][4 * top_xy + 2]];
            rc[2 - 8] = rc[3 - 8] = r2f[h->cur_pic.ref_index[list][4 * top_xy + 3]];
        } else {
            memset(mv - 8, 0, 16);
            memset(rc - 8, LIST_NOT_USED, 4);
        }
        if (USES_LIST(left_type, list)) {                        /* right 4x4 column of the MB to the left */
            const int *r2f = &h->ref2frm[h->slice_table[left_xy] & (MAX_SLICES - 1)][list][2];
            const int b_xy = h->mb2b_xy[left_xy] + 3;
            for (i = 0; i < 4; i++) {
                memcpy(mv - 1 + 8 * i, h->cur_pic.motion_val[list][b_xy + bs * i], 4);
                rc[-1 + 8 * i] = r2f[h->cur_pic.ref_index[list][4 * left_xy + 1 + 2 * (i >> 1)]];
            }
        } else {
            for (i = 0; i < 4; i++) { memset(mv - 1 + 8 * i, 0, 4); rc[-1 + 8 * i] = LIST_NOT_USED; }
        }
    }
    if (!USES_LIST(mb_type, list)) {
        for (r = 0; r < 4; r++) { memset(mv + 8 * r, 0, 16); memset(rc + 8 * r, LIST_NOT_USED, 4); }
        return;
    }
    {
        const int8_t *ref = &h->cur_pic.ref_index[list][4 * mb_xy];
        const int *r2f = &h->ref2frm[sl->slice_num & (MAX_SLICES - 1)][list][2];
        const int16_t (*src)[2] = &h->cur_pic.motion_val[list][4 * sl->mb_x + 4 * sl->mb_y * bs];
        for (r = 0; r < 4; r++) {
            rc[8 * r + 0] = rc[8 * r + 1] = r2f[ref[2 * (r >> 1)]];
            rc[8 * r + 2] = rc[8 * r + 3] = r2f[ref[2 * (r >> 1) + 1]];
            memcpy(mv + 8 * r, src + r * bs, 16);
        }
    }
}

/* returns 1 when the macroblock is skipped by the qp threshold shortcut (h264_slice.c:2085-2107) */
static int gather_caches(const H264Context *h, H264SliceContext *sl, int mb_type)
{
    const int mb_xy = sl->mb_xy, top_xy = mb_xy - h->mb_stride, left_xy = mb_xy - 1;
    const int qp = h->cur_pic.qscale_table[mb_xy], th = sl->qp_thresh;
    int top_type, left_type, r, k;
    uint8_t *nc = sl->non_zero_count_cache;
    sl->top_mb_xy = top_xy;
    sl->left_mb_xy[LTOP] = sl->left_mb_xy[LBOT] = left_xy;
    if (qp <= th && (left_xy < 0 || ((qp + h->cur_pic.qscale_table[left_xy] + 1) >> 1) <= th) &&
                    (top_xy  < 0 || ((qp + h->cur_pic.qscale_table[top_xy]  + 1) >> 1) <= th))
        return 1;
    top_type  = h->cur_pic.mb_type[top_xy];
    left_type = h->cur_pic.mb_type[left_xy];
    if (sl->deblocking_filter == 2) {
        if (h->slice_table[top_xy]  != sl->slice_num) top_type  = 0;
        if (h->slice_table[left_xy] != sl->slice_num) left_type = 0;
    } else {
        if (h->slice_table[top_xy]  == 0xFFFF) top_type  = 0;
        if (h->slice_table[left_xy] == 0xFFFF) left_type = 0;
    }
    sl->top_type = top_type;
    sl->left_type[LTOP] = sl->left_type[LBOT] = left_type;
    if (IS_INTRA(mb_type))
        return 0;
    gather_list(h, sl, mb_type, top_xy, left_xy, top_type, left_type, mb_xy, 0);
    if (sl->list_count == 2)
        gather_list(h, sl, mb_type, top_xy, left_xy, top_type, left_type, mb_xy, 1);
    for (r = 0; r < 4; r++)
        memcpy(&nc[4 + 8 * (r + 1)], &h->non_zero_count[mb_xy][4 * r], 4);
    sl->cbp = h->cbp_table[mb_xy];
    if (top_type)
        memcpy(&nc[4], &h->non_zero_count[top_xy][12], 4);
    if (left_type)
        for (r = 0; r < 4; r++) nc[3 + 8 * (r + 1)] = h->non_zero_count[left_xy][3 + 4 * r];
    if (!h->ps.pps->cabac && h->ps.pps->transform_8x8_mode) {    /* CAVLC keeps per-8x8 flags in cbp_table bits 12..15 */
        if (IS_8x8DCT(top_type)) {
            nc[4] = nc[5] = (h->cbp_table[top_xy] & 0x4000) >> 12;
            nc[6] = nc[7] = (h->cbp_table[top_xy] & 0x8000) >> 12;
        }
        if (IS_8x8DCT(left_type)) {
            nc[3 + 8 * 1] = nc[3 + 8 * 2] = (h->cbp_table[left_xy] & 0x2000) >> 12;
            nc[3 + 8 * 3] = nc[3 + 8 * 4] = (h->cbp_table[left_xy] & 0x8000) >> 12;
        }
        if (IS_8x8DCT(mb_type))
            for (k = 0; k < 16; k++) nc[scan8[k]] = (sl->cbp & (0x1000 << (k >> 2))) >> 12;
    }
    return 0;
}

/* PAFF field pictures: h->picture_structure for the pictures that follow (the caller's mb_type entries then carry MB_TYPE_INTERLACED, as
 * ff_h264_decode_mb_* leave them in a field picture); MBAFF is not driven */
static int g_field_picture;
void ref_h264_deblock_picture_structure(int field_picture) { g_field_picture = field_picture != 0; }

/* table == NULL: the recorders above (decisions into `out`).  table != NULL: an H264DSPContext whose loop-filter entries are called on the
 * real picture planes Y / Cb / Cr (pitches ls / uvls) with the pointers loop_filter() passes (h264_slice.c:2198-2262), `out` unused. */
static int run_driver(const H264DSPContext *table, uint8_t *Y, uint8_t *Cb, uint8_t *Cr, int ls, int uvls,
                      int mb_w, int mb_h, const uint32_t *mb_type, const int8_t *qscale, const uint8_t *nnz,
                      const uint16_t *cbp, const uint16_t *slice_table, const int16_t *mv0, const int16_t *mv1,
                      const int8_t *ref0, const int8_t *ref1, const int32_t *slice_params, int n_slices,
                      const uint8_t *chroma_qp_table, int cabac, int transform_8x8_mode, int bit_depth, uint8_t *out)
{
    const int ms = mb_w + 1, pad = 2 * ms + 1, n = ms * mb_h;
    H264Context *h = calloc(1, sizeof(*h));
    H264SliceContext *sl = calloc(1, sizeof(*sl));
    PPS *pps = calloc(1, sizeof(*pps));
    SPS *sps = calloc(1, sizeof(*sps));
    /* padded copies: the reference reads mb_xy - 1 and mb_xy - mb_stride of border macroblocks */
    uint32_t *t_type  = calloc(n + pad, sizeof(*t_type));
    int8_t   *t_qp    = calloc(n + pad, 1);
    uint16_t *t_slice = malloc((n + pad) * sizeof(*t_slice));
    uint16_t *t_cbp   = calloc(n + pad, sizeof(*t_cbp));
    uint8_t (*t_nnz)[48] = calloc(n + pad, 48);
    int8_t   *t_ref[2];
    uint32_t *t_b = calloc(n + pad, sizeof(*t_b));
    int x, y, s, l;
    if (n_slices > MAX_SLICES) return -1;
    memset(t_slice, 0xFF, (n + pad) * sizeof(*t_slice));
    for (l = 0; l < 2; l++) t_ref[l] = calloc(4 * (n + pad), 1);
    for (y = 0; y < mb_h; y++)
        for (x = 0; x < mb_w; x++) {
            const int xy = x + y * ms;
            t_type[pad + xy] = mb_type[xy]; t_qp[pad + xy] = qscale[xy]; t_slice[pad + xy] = slice_table[xy];
            t_cbp[pad + xy] = cbp[xy]; memcpy(t_nnz[pad + xy], nnz + 48 * xy, 48);
            memcpy(t_ref[0] + 4 * (pad + xy), ref0 + 4 * xy, 4);
            memcpy(t_ref[1] + 4 * (pad + xy), ref1 + 4 * xy, 4);
            t_b[pad + xy] = 4 * x + 4 * y * 4 * mb_w;
        }
    h->mb_width = mb_w; h->mb_height = mb_h; h->mb_stride = ms; h->b_stride = 4 * mb_w;
    h->cur_pic.mb_type = t_type + pad; h->cur_pic.qscale_table = t_qp + pad;
    h->slice_table = t_slice + pad; h->cbp_table = t_cbp + pad; h->non_zero_count = t_nnz + pad;
    h->mb2b_xy = t_b + pad;
    h->cur_pic.motion_val[0] = (int16_t (*)[2])mv0; h->cur_pic.motion_val[1] = (int16_t (*)[2])mv1;
    h->cur_pic.ref_index[0] = t_ref[0] + 4 * pad; h->cur_pic.ref_index[1] = t_ref[1] + 4 * pad;
    h->picture_structure = g_field_picture ? PICT_TOP_FIELD : PICT_FRAME;
    pps->cabac = cabac; pps->transform_8x8_mode = transform_8x8_mode;
    memcpy(pps->chroma_qp_table, chroma_qp_table, 128);
    pps->chroma_qp_diff = memcmp(chroma_qp_table, chroma_qp_table + 64, 64) != 0;
    /* bit_depth_luma sets qp_bd_offset (h264_loopfilter.c:256,726); the recorders keep pixel_shift 0, so offsets into the fake planes still
     * name the edge, while real 9 / 10-bit planes hold 16-bit samples */
    sps->bit_depth_luma = bit_depth; sps->chroma_format_idc = (g_ext422 && !table) ? 2 : 1;
    h->pixel_shift = table && bit_depth > 8;
    h->ps.pps = pps; h->ps.sps = sps;
    for (s = 0; s < n_slices; s++)
        memcpy(h->ref2frm[s], slice_params + 133 * s + 5, sizeof(h->ref2frm[s]));
    h->h264dsp.h264_h_loop_filter_luma         = r_h_luma;     h->h264dsp.h264_v_loop_filter_luma         = r_v_luma;
    h->h264dsp.h264_h_loop_filter_luma_intra   = r_h_luma_i;   h->h264dsp.h264_v_loop_filter_luma_intra   = r_v_luma_i;
    h->h264dsp.h264_h_loop_filter_chroma       = r_h_chroma;   h->h264dsp.h264_v_loop_filter_chroma       = r_v_chroma;
    h->h264dsp.h264_h_loop_filter_chroma_intra = r_h_chroma_i; h->h264dsp.h264_v_loop_filter_chroma_intra = r_v_chroma_i;
    h->h264dsp.h264_loop_filter_strength = NULL;               /* what ff_h264dsp_init leaves in the C build */
    if (table) h->h264dsp = *table;

    if (!table) memset(out, 0, (size_t)104 * mb_w * mb_h);
    if (!table && g_ext422) memset(g_ext422, 0, (size_t)52 * mb_w * mb_h);
    for (y = 0; y < mb_h; y++)
        for (x = 0; x < mb_w; x++) {
            const int xy = x + y * ms, type = h->cur_pic.mb_type[xy];
            const int32_t *sp = slice_params + 133 * h->slice_table[xy];
            if (!table) { cur_rec = out + (size_t)104 * (x + y * mb_w); cur_ext = g_ext422 ? g_ext422 + (size_t)52 * (x + y * mb_w) : NULL; }
            sl->mb_xy = xy; sl->mb_x = x; sl->mb_y = y;
            sl->slice_num = h->slice_table[xy];
            sl->slice_alpha_c0_offset = sp[0]; sl->slice_beta_offset = sp[1];
            sl->deblocking_filter = sp[2]; sl->list_count = sp[3]; sl->qp_thresh = sp[4];
            if (!sl->deblocking_filter || gather_caches(h, sl, type))
                continue;
            sl->chroma_qp[0] = pps->chroma_qp_table[0][h->cur_pic.qscale_table[xy] & 63];
            sl->chroma_qp[1] = pps->chroma_qp_table[1][h->cur_pic.qscale_table[xy] & 63];
            if (table) ff_h264_filter_mb_fast(h, sl, x, y, Y + (16 * x << h->pixel_shift) + 16 * (size_t)y * ls, Cb + (8 * x << h->pixel_shift) + 8 * (size_t)y * uvls,
                                              Cr + (8 * x << h->pixel_shift) + 8 * (size_t)y * uvls, ls, uvls);
            else       ff_h264_filter_mb_fast(h, sl, x, y, fake_y, fake_cb, fake_cr, REC_LS, REC_UVLS);
        }
    for (l = 0; l < 2; l++) free(t_ref[l]);
    free(t_b); free(t_nnz); free(t_cbp); free(t_slice); free(t_qp); free(t_type); free(sps); free(pps); free(sl); free(h);
    return 0;
}

/* bit_depth 8 / 9 / 10 (-1 otherwise); ref_h264_deblock_params keeps its 8-bit signature */
int ref_h264_deblock_params_hbd(int bit_depth, int mb_w, int mb_h, const uint32_t *mb_type, const int8_t *qscale, const uint8_t *nnz,
                                const uint16_t *cbp, const uint16_t *slice_table, const int16_t *mv0, const int16_t *mv1,
                                const int8_t *ref0, const int8_t *ref1, const int32_t *slice_params, int n_slices,
                                const uint8_t *chroma_qp_table, int cabac, int transform_8x8_mode, uint8_t *out)
{
    if (bit_depth < 8 || bit_depth > 10) return -1;
    return run_driver(NULL, NULL, NULL, NULL, 0, 0, mb_w, mb_h, mb_type, qscale, nnz, cbp, slice_table, mv0, mv1, ref0, ref1, slice_params, n_slices,
                      chroma_qp_table, cabac, transform_8x8_mode, bit_depth, out);
}

int ref_h264_deblock_params(int mb_w, int mb_h, const uint32_t *mb_type, const int8_t *qscale, const uint8_t *nnz,
                            const uint16_t *cbp, const uint16_t *slice_table, const int16_t *mv0, const int16_t *mv1,
                            const int8_t *ref0, const int8_t *ref1, const int32_t *slice_params, int n_slices,
                            const uint8_t *chroma_qp_table, int cabac, int transform_8x8_mode, uint8_t *out)
{
    return ref_h264_deblock_params_hbd(8, mb_w, mb_h, mb_type, qscale, nnz, cbp, slice_table, mv0, mv1, ref0, ref1, slice_params, n_slices,
                                       chroma_qp_table, cabac, transform_8x8_mode, out);
}

/* The reference's own deblocking driver (ff_h264_filter_mb_fast -> ff_h264_filter_mb, raster order like loop_filter()) filtering a real
 * picture in place through the loop-filter entries of `table` -- an H264DSPContext filled by anybody: NULL = ff_h264dsp_init(bit_depth, 1),
 * the reference's C functions; otherwise e.g. the table ff_h264dsp_init_cuda() filled (tests/h264_dropin_cases.py).  At 9 / 10 bit the
 * planes hold uint16 samples and ls / uvls count bytes; ref_h264_deblock_picture_with is the 8-bit call.  Only in _ref. */
int ref_h264_deblock_picture_with_hbd(int bit_depth, const void *table, uint8_t *Y, uint8_t *Cb, uint8_t *Cr, int ls, int uvls,
                                      int mb_w, int mb_h, const uint32_t *mb_type, const int8_t *qscale, const uint8_t *nnz,
                                      const uint16_t *cbp, const uint16_t *slice_table, const int16_t *mv0, const int16_t *mv1,
                                      const int8_t *ref0, const int8_t *ref1, const int32_t *slice_params, int n_slices,
                                      const uint8_t *chroma_qp_table, int cabac, int transform_8x8_mode)
{
    H264DSPContext c_table;
    if (bit_depth < 8 || bit_depth > 10) return -1;
    if (!table) { ff_h264dsp_init(&c_table, bit_depth, 1); table = &c_table; }
    return run_driver(table, Y, Cb, Cr, ls, uvls, mb_w, mb_h, mb_type, qscale, nnz, cbp, slice_table, mv0, mv1, ref0, ref1, slice_params, n_slices,
                      chroma_qp_table, cabac, transform_8x8_mode, bit_depth, NULL);
}

int ref_h264_deblock_picture_with(const void *table, uint8_t *Y, uint8_t *Cb, uint8_t *Cr, int ls, int uvls,
                                  int mb_w, int mb_h, const uint32_t *mb_type, const int8_t *qscale, const uint8_t *nnz,
                                  const uint16_t *cbp, const uint16_t *slice_table, const int16_t *mv0, const int16_t *mv1,
                                  const int8_t *ref0, const int8_t *ref1, const int32_t *slice_params, int n_slices,
                                  const uint8_t *chroma_qp_table, int cabac, int transform_8x8_mode)
{
    return ref_h264_deblock_picture_with_hbd(8, table, Y, Cb, Cr, ls, uvls, mb_w, mb_h, mb_type, qscale, nnz, cbp, slice_table, mv0, mv1, ref0, ref1,
                                             slice_params, n_slices, chroma_qp_table, cabac, transform_8x8_mode);
}
