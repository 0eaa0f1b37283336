/*
 * oracle/port/orc_h264lf.c -- TEST INFRASTRUCTURE, NOT PRODUCT.
 *
 * CPU restatement of the H.264 deblocking DECISIONS for progressive 4:2:0 / 4:2:2 pictures at 8, 9 or 10 bit: boundary strength per
 * 4-sample edge segment and the (alpha, beta, tc0) each edge is filtered with, i.e. what
 *   loop_filter() / fill_filter_caches()           libavcodec/h264_slice.c:1972-2262
 *   ff_h264_filter_mb() / filter_mb_dir() / check_mv()  libavcodec/h264_loopfilter.c:438-846
 *   filter_mb_edge{v,h,cv,ch}()                    libavcodec/h264_loopfilter.c:103-236
 * hand to the H264DSPContext loop-filter slots.  Written from the picture-level arrays directly (no per-macroblock
 * caches): strength(dir, edge, i) looks the two 4x4 blocks of segment i up where they live.  The threshold tables
 * are the standard's alpha'/beta'/tC0' with the index clipped to 0..51, which is what the reference's zero-/
 * constant-padded tables (:40-101) evaluate to.  At 9 / 10 bit qscale_table and chroma_qp_table hold QP' (0..51 + qp_bd_offset, the
 * decoder's scale); only the table index subtracts qp_bd_offset = 6 * (bit_depth - 8) (:256-258,726-728), the qp averaging and the
 * low-qp shortcut stay in QP'.  Pinned byte-for-byte against oracle/_ref (the reference's own
 * h264_loopfilter.c with recording slots) in tests/test_oracle_h264lf_cpu.py.
 */
#include <stdint.h>
#include <string.h>
#include "../oracle_api.h"

enum { T_INTRA = 7, T_16x16 = 8, T_16x8 = 16, T_8x16 = 32, T_INTERLACED = 0x80, T_DCT8 = 0x01000000 };

/* h->picture_structure != PICT_FRAME for the pictures that follow (PAFF field pictures: every macroblock type carries MB_TYPE_INTERLACED) */
static int g_field_picture;
void orc_h264_deblock_picture_structure(int field_picture) { g_field_picture = field_picture != 0; }
/* chroma_format_idc 2: the horizontal chroma edges (four per macroblock: chroma rows 0, 4, 8, 12 of the 8 x 16 block, one per luma edge,
 * h264_loopfilter.c:633,693-700) go to a second record per macroblock, 52 bytes: alpha[2 planes][4], beta[2][4], tc0[2][4][4], intra[2], pad[2];
 * the vertical ones keep the 4:2:0 fields (each tc0 entry then covers four of the sixteen lines) */
static uint8_t *g_ext422;
void orc_h264_deblock_chroma422(uint8_t *ext) { g_ext422 = ext; }
static int g_ylim = 4;          /* mvy_limit of the macroblock being decided (h264_loopfilter.c:723) */
#define USES(t, l) ((t) & (0x3000 << (2 * (l))))

static const uint8_t alpha_std[52] = {
    0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 4, 4, 5, 6, 7, 8, 9, 10, 12, 13, 15, 17, 20, 22, 25, 28,
    32, 36, 40, 45, 50, 56, 63, 71, 80, 90, 101, 113, 127, 144, 162, 182, 203, 226, 255, 255 };
static const uint8_t beta_std[52] = {
    0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 2, 2, 2, 3, 3, 3, 3, 4, 4, 4, 6, 6, 7, 7, 8, 8,
    9, 9, 10, 10, 11, 11, 12, 12, 13, 13, 14, 14, 15, 15, 16, 16, 17, 17, 18, 18 };
static const uint8_t tc0_std[52][3] = {
    {0,0,0},{0,0,0},{0,0,0},{0,0,0},{0,0,0},{0,0,0},{0,0,0},{0,0,0},{0,0,0},{0,0,0},{0,0,0},{0,0,0},{0,0,0},{0,0,0},
    {0,0,0},{0,0,0},{0,0,0},{0,0,1},{0,0,1},{0,0,1},{0,0,1},{0,1,1},{0,1,1},{1,1,1},{1,1,1},{1,1,1},{1,1,1},{1,1,2},
    {1,1,2},{1,1,2},{1,1,2},{1,2,3},{1,2,3},{2,2,3},{2,2,4},{2,3,4},{2,3,4},{3,3,5},{3,4,6},{3,4,6},{4,5,7},{4,5,8},
    {4,6,9},{5,7,10},{6,8,11},{6,8,13},{7,10,14},{8,11,16},{9,12,18},{10,13,20},{11,15,23},{13,17,25} };

typedef struct Pic {
    int mb_w, mb_h, ms, bs, cabac, t8x8;
    const uint32_t *type; const int8_t *qp; const uint8_t *nnz; const uint16_t *cbp, *slice;
    const int16_t *mv[2]; const int8_t *ref[2]; const int32_t *sp; const uint8_t *cqp;
} Pic;

typedef struct Blk { int nz; int ref[2]; int mvx[2], mvy[2]; } Blk;

/* one 4x4 block (bx, by) of macroblock (x, y) as the loop filter sees it; `type` is the macroblock's type after
 * the availability masking (0 = treat every list as unused) */
static Blk block_of(const Pic *p, int x, int y, int bx, int by, uint32_t type, int cavlc8_kind)
{
    const int xy = x + y * p->ms;
    Blk b;
    b.nz = p->nnz[48 * xy + bx + 4 * by];
    if (!p->cabac && p->t8x8 && (p->type[xy] & T_DCT8)) {
        /* CAVLC 8x8 transform: per-8x8 flags of cbp_table bits 12..15 replace the counts (h264_slice.c:2155-2193);
         * the left neighbour's upper half reads bit 13 where the own-MB rule would read bit 12 (reference behaviour) */
        const int cbp = p->cbp[xy];
        if (cavlc8_kind == 0)      b.nz = (cbp & (0x1000 << ((bx >> 1) + 2 * (by >> 1)))) >> 12;     /* own MB */
        else if (cavlc8_kind == 1) b.nz = (cbp & (bx < 2 ? 0x4000 : 0x8000)) >> 12;                  /* MB above */
        else                       b.nz = (cbp & (by < 2 ? 0x2000 : 0x8000)) >> 12;                  /* MB to the left */
    }
    for (int l = 0; l < 2; l++) {
        if (USES(type, l)) {
            const int32_t *r2f = p->sp + 133 * (p->slice[xy] & 31) + 5 + 64 * l + 2;
            b.ref[l] = (int8_t)r2f[p->ref[l][4 * xy + (bx >> 1) + 2 * (by >> 1)]];
            const int16_t *m = p->mv[l] + 2 * ((4 * x + bx) + (4 * y + by) * p->bs);
            b.mvx[l] = m[0]; b.mvy[l] = m[1];
        } else {
            b.ref[l] = -1; b.mvx[l] = b.mvy[l] = 0;
        }
    }
    return b;
}

static int far(int a, int b) { int d = a - b; return d >= 4 || d <= -4; }
static int far_y(int a, int b) { int d = a - b; return d >= g_ylim || d <= -g_ylim; }

/* check_mv(), h264_loopfilter.c:438-469 */
static int motion_differs(const Blk *a, const Blk *b, int list_count)
{
    int v = a->ref[0] != b->ref[0];
    if (!v && a->ref[0] != -1)
        v = far(a->mvx[0], b->mvx[0]) | far_y(a->mvy[0], b->mvy[0]);
    if (list_count == 2) {
        if (!v)
            v = (a->ref[1] != b->ref[1]) | far(a->mvx[1], b->mvx[1]) | far_y(a->mvy[1], b->mvy[1]);
        if (v) {
            if ((a->ref[0] != b->ref[1]) | (a->ref[1] != b->ref[0]))
                return 1;
            return far(a->mvx[0], b->mvx[1]) | far_y(a->mvy[0], b->mvy[1]) | far(a->mvx[1], b->mvx[0]) | far_y(a->mvy[1], b->mvy[0]);
        }
    }
    return v;
}

static int idx51(int v) { return v < 0 ? -1 : v > 51 ? 51 : v; }

/* filter_mb_edge*: write one edge's parameters; chroma = 0 luma, 1 cb, 2 cr */
static void emit(uint8_t *rec, int chroma, int dir, int e, const int bS[4], int qp, int offa, int offb, int may_be_intra)
{
    const int ia = idx51(qp + offa), ib = idx51(qp + offb);
    const int alpha = ia < 0 ? 0 : alpha_std[ia], beta = ib < 0 ? 0 : beta_std[ib];
    if (!alpha || !beta) return;
    uint8_t *pa, *pb, *pi; int8_t *pt; int bit;
    if (!chroma) { pa = rec + 0 + 4 * dir + e; pb = rec + 8 + 4 * dir + e; pt = (int8_t *)rec + 16 + 16 * dir + 4 * e; pi = rec + 48 + dir; bit = e; }
    else {
        const int i = ((chroma - 1) * 2 + dir) * 2 + (e >> 1);
        pa = rec + 50 + i; pb = rec + 58 + i; pt = (int8_t *)rec + 66 + 4 * i; pi = rec + 98 + (chroma - 1) * 2 + dir; bit = e >> 1;
    }
    *pa = alpha; *pb = beta;
    if (bS[0] < 4 || !may_be_intra)
        for (int i = 0; i < 4; i++) pt[i] = (bS[i] ? (int)tc0_std[ia][bS[i] - 1] : -1) + (chroma ? 1 : 0);
    else
        *pi |= 1 << bit;
}
/* a horizontal chroma edge of a 4:2:2 macroblock -> the extension record */
static void emit422(uint8_t *ext, int plane, int e, const int bS[4], int qp, int offa, int offb, int may_be_intra)
{
    const int ia = idx51(qp + offa), ib = idx51(qp + offb);
    const int alpha = ia < 0 ? 0 : alpha_std[ia], beta = ib < 0 ? 0 : beta_std[ib];
    if (!alpha || !beta) return;
    ext[4 * plane + e] = alpha; ext[8 + 4 * plane + e] = beta;
    int8_t *pt = (int8_t *)ext + 16 + 16 * plane + 4 * e;
    if (bS[0] < 4 || !may_be_intra)
        for (int i = 0; i < 4; i++) pt[i] = (bS[i] ? (int)tc0_std[ia][bS[i] - 1] : -1) + 1;
    else
        ext[48 + plane] |= 1 << e;
}

int orc_h264_deblock_params_hbd(int bit_depth, int mb_w, int mb_h, const uint32_t *mb_type, const int8_t *qscale, const uint8_t *nnz,
                                const uint16_t *cbp, const uint16_t *slice_table, const int16_t *mv0, const int16_t *mv1,
                                const int8_t *ref0, const int8_t *ref1, const int32_t *slice_params, int n_slices,
                                const uint8_t *chroma_qp_table, int cabac, int transform_8x8_mode, uint8_t *out)
{
    static const uint8_t mask_edge_tab[2][8] = { { 0, 3, 3, 3, 1, 1, 1, 1 }, { 0, 3, 1, 1, 3, 3, 3, 3 } };
    Pic p = { mb_w, mb_h, mb_w + 1, 4 * mb_w, cabac, transform_8x8_mode, mb_type, qscale, nnz, cbp, slice_table,
              { mv0, mv1 }, { ref0, ref1 }, slice_params, chroma_qp_table };
    if (n_slices > 32 || bit_depth < 8 || bit_depth > 10) return -1;
    const int qp_bd_offset = 6 * (bit_depth - 8);
    memset(out, 0, (size_t)104 * mb_w * mb_h);
    if (g_ext422) memset(g_ext422, 0, (size_t)52 * mb_w * mb_h);
    for (int y = 0; y < mb_h; y++)
        for (int x = 0; x < mb_w; x++) {
            const int xy = x + y * p.ms, sn = slice_table[xy];
            uint8_t *ext = g_ext422 ? g_ext422 + (size_t)52 * (x + y * mb_w) : NULL;
            const int32_t *sp = slice_params + 133 * sn;
            /* offa / offb reach only the table index inside emit / emit422: the reference's a = 52 + offset - qp_bd_offset */
            const int offa = sp[0] - qp_bd_offset, offb = sp[1] - qp_bd_offset, mode = sp[2], lists = sp[3], th = sp[4];
            const uint32_t type = mb_type[xy];
            const int qp = qscale[xy];
            uint8_t *rec = out + (size_t)104 * (x + y * mb_w);
            if (!mode) continue;
            /* low-qp shortcut (h264_slice.c:2085-2107): the reference's index arithmetic makes the left neighbour
             * of column 0 the zero-initialised padding entry of the row above, except for the very first MB */
            {
                const int has_l = xy - 1 >= 0, has_t = xy - p.ms >= 0;
                const int ql = x > 0 ? qscale[xy - 1] : 0, qt = y > 0 ? qscale[xy - p.ms] : 0;
                if (qp <= th && (!has_l || ((qp + ql + 1) >> 1) <= th) && (!has_t || ((qp + qt + 1) >> 1) <= th))
                    continue;
            }
            uint32_t ntype[2];                                   /* [0] left, [1] top; 0 = not available */
            ntype[0] = x > 0 ? mb_type[xy - 1] : 0;
            ntype[1] = y > 0 ? mb_type[xy - p.ms] : 0;
            if (mode == 2) {
                if (x > 0 && slice_table[xy - 1] != sn) ntype[0] = 0;
                if (y > 0 && slice_table[xy - p.ms] != sn) ntype[1] = 0;
            }
            const int cq[2] = { chroma_qp_table[qp], chroma_qp_table[64 + qp] };
            for (int dir = 0; dir < 2; dir++) {
                const int nx = dir ? x : x - 1, ny = dir ? y - 1 : y;
                const uint32_t mt = ntype[dir];
                const int mask_edge = mask_edge_tab[dir][(type >> 3) & 7];
                const int luma_cbp = (type & T_INTRA) ? 0 : cbp[xy] & 15;
                const int edges = (mask_edge == 3 && !luma_cbp && !(type & T_INTRA)) ? 1 : 4;
                const uint32_t par0 = type & (T_16x16 | (T_8x16 >> dir));
                for (int e = 0; e < edges; e++) {
                    int bS[4], sum = 0;
                    if (e == 0 && !mt) continue;
                    const int deblock_edge = !(e && (type & T_DCT8) && (e & 1));     /* inside an 8x8 transform block: no luma edge; 4:2:2 chroma still has one (:633) */
                    if (!deblock_edge && !(ext && dir == 1)) continue;
                    g_ylim = (type & T_INTERLACED) ? 2 : 4;
                    if (e == 0 && ((type | mt) & T_INTRA)) {
                        /* 3 across the horizontal macroblock edges of a field picture, 4 otherwise (h264_loopfilter.c:551-557) */
                        bS[0] = bS[1] = bS[2] = bS[3] = (((type | mt) & T_INTERLACED) && !(g_field_picture && dir == 0)) ? 3 : 4;
                    } else if (type & T_INTRA) {
                        bS[0] = bS[1] = bS[2] = bS[3] = 3;
                    } else {
                        int whole = -1;                          /* one motion decision for the whole edge */
                        if (e && (e & mask_edge)) whole = 0;
                        else if (par0 && (e || (mt & (T_16x16 | (T_8x16 >> dir))))) {
                            Blk a = block_of(&p, x, y, dir ? 0 : e, dir ? e : 0, type, 0);
                            Blk b = e ? block_of(&p, x, y, dir ? 0 : e - 1, dir ? e - 1 : 0, type, 0)
                                      : block_of(&p, nx, ny, dir ? 0 : 3, dir ? 3 : 0, mt, dir ? 1 : 2);
                            whole = motion_differs(&a, &b, lists);
                        }
                        for (int i = 0; i < 4; i++) {
                            const int bx = dir ? i : e, by = dir ? e : i;
                            Blk a = block_of(&p, x, y, bx, by, type, 0);
                            Blk b = e ? block_of(&p, x, y, dir ? i : e - 1, dir ? e - 1 : i, type, 0)
                                      : block_of(&p, nx, ny, dir ? i : 3, dir ? 3 : i, mt, dir ? 1 : 2);
                            bS[i] = (a.nz | b.nz) ? 2 : whole >= 0 ? whole : motion_differs(&a, &b, lists);
                        }
                    }
                    for (int i = 0; i < 4; i++) sum += bS[i];
                    if (!sum) continue;
                    if (e == 0) {
                        const int qn = qscale[nx + ny * p.ms];
                        const int qa0 = (cq[0] + chroma_qp_table[qn] + 1) >> 1, qa1 = (cq[1] + chroma_qp_table[64 + qn] + 1) >> 1;
                        emit(rec, 0, dir, 0, bS, (qp + qn + 1) >> 1, offa, offb, 1);
                        if (ext && dir == 1) { emit422(ext, 0, 0, bS, qa0, offa, offb, 1); emit422(ext, 1, 0, bS, qa1, offa, offb, 1); }
                        else { emit(rec, 1, dir, 0, bS, qa0, offa, offb, 1); emit(rec, 2, dir, 0, bS, qa1, offa, offb, 1); }
                    } else {
                        if (deblock_edge) emit(rec, 0, dir, e, bS, qp, offa, offb, 0);
                        if (ext && dir == 1) { emit422(ext, 0, e, bS, cq[0], offa, offb, 0); emit422(ext, 1, e, bS, cq[1], offa, offb, 0); }
                        else if (!(e & 1)) { emit(rec, 1, dir, e, bS, cq[0], offa, offb, 0); emit(rec, 2, dir, e, bS, cq[1], offa, offb, 0); }
                    }
                }
            }
        }
    return 0;
}

int orc_h264_deblock_params(int mb_w, int mb_h, const uint32_t *mb_type, const int8_t *qscale, const uint8_t *nnz,
                            const uint16_t *cbp, const uint16_t *slice_table, const int16_t *mv0, const int16_t *mv1,
                            const int8_t *ref0, const int8_t *ref1, const int32_t *slice_params, int n_slices,
                            const uint8_t *chroma_qp_table, int cabac, int transform_8x8_mode, uint8_t *out)
{
    return orc_h264_deblock_params_hbd(8, mb_w, mb_h, mb_type, qscale, nnz, cbp, slice_table, mv0, mv1, ref0, ref1, slice_params, n_slices,
                                       chroma_qp_table, cabac, transform_8x8_mode, out);
}
