// libav_b200/csrc/h264lf.cu -- H.264 deblocking DECISIONS on the device (SURVEY 8f rank 1).
//
// Replaces the per-macroblock scalar walk loop_filter() -> fill_filter_caches() -> ff_h264_filter_mb()
// (libavcodec/h264_slice.c:1972-2262, libavcodec/h264_loopfilter.c:438-846) for progressive 4:2:0 8-bit pictures:
// from the decoder's side-information arrays (device copies, the decoder's own layouts) it writes one FFH264DeblockMB
// per macroblock -- the (alpha, beta, tc0 | bS 4) of every edge -- which ff_h264_deblock_batch_cuda consumes without
// a host round trip.  One thread = one (macroblock, direction): it owns every field of the record indexed by that
// direction, so no two threads write the same byte.  Neighbour blocks are read where they live (no cache gather).
#include "common.cuh"
#include "../../include/avdsp_b200.h"

namespace avb {

__constant__ uint8_t c_alpha[52] = {
    0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 4, 4, 5, 6, 7, 8, 9, 10, 12, 13, 15, 17, 20, 22, 25, 28,
    32, 36, 40, 45, 50, 56, 63, 71, 80, 90, 101, 113, 127, 144, 162, 182, 203, 226, 255, 255 };
__constant__ uint8_t c_beta[52] = {
    0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 2, 2, 2, 3, 3, 3, 3, 4, 4, 4, 6, 6, 7, 7, 8, 8,
    9, 9, 10, 10, 11, 11, 12, 12, 13, 13, 14, 14, 15, 15, 16, 16, 17, 17, 18, 18 };
// tC0' for bS 1..3 (the reference's tc0_table rows minus the -1 of bS 0, h264_loopfilter.c:66-101)
__constant__ uint8_t c_tc0[52][3] = {
    {0,0,0},{0,0,0},{0,0,0},{0,0,0},{0,0,0},{0,0,0},{0,0,0},{0,0,0},{0,0,0},{0,0,0},{0,0,0},{0,0,0},{0,0,0},{0,0,0},
    {0,0,0},{0,0,0},{0,0,0},{0,0,1},{0,0,1},{0,0,1},{0,0,1},{0,1,1},{0,1,1},{1,1,1},{1,1,1},{1,1,1},{1,1,1},{1,1,2},
    {1,1,2},{1,1,2},{1,1,2},{1,2,3},{1,2,3},{2,2,3},{2,2,4},{2,3,4},{2,3,4},{3,3,5},{3,4,6},{3,4,6},{4,5,7},{4,5,8},
    {4,6,9},{5,7,10},{6,8,11},{6,8,13},{7,10,14},{8,11,16},{9,12,18},{10,13,20},{11,15,23},{13,17,25} };

enum : uint32_t { T_INTRA = 7, T_16x16 = 8, T_8x16 = 32, T_INTERLACED = 0x80, T_DCT8 = 0x01000000 };
__device__ __forceinline__ uint32_t uses_list(uint32_t t, int l) { return t & (0x3000u << (2 * l)); }

struct Blk { int nz, ref0, ref1; int mv0, mv1; };          // mv = packed (x, y) int16 pair

struct LfPic {
    FFH264DeblockInfo i;
    int ms, bs;
};

// the 4x4 block (bx, by) of macroblock xy (picture-stacked index) as the loop filter sees it; `type` = macroblock
// type after availability masking; kind 0 own / 1 above / 2 left selects the CAVLC 8x8 flag rule (h264_slice.c:2155-2193)
__device__ __forceinline__ Blk fetch_block(const LfPic &p, int xy, int bx4, int by4, int bx, int by, uint32_t type, int kind)
{
    Blk b;
    b.nz = p.i.non_zero_count[48 * (size_t)xy + bx + 4 * by];
    if (!p.i.cabac && p.i.transform_8x8_mode && (p.i.mb_type[xy] & T_DCT8)) {
        const int cbp = p.i.cbp_table[xy];
        b.nz = kind == 0 ? (cbp >> (12 + (bx >> 1) + 2 * (by >> 1))) & 1
             : kind == 1 ? cbp & (bx < 2 ? 0x4000 : 0x8000)
                         : cbp & (by < 2 ? 0x2000 : 0x8000);
    }
    const int32_t *r2f = p.i.slices[p.i.slice_table[xy] & 31].ref2frm[0];
    const int b8 = (bx >> 1) + 2 * (by >> 1);
    const size_t mvi = (size_t)(bx4 + bx) + (size_t)(by4 + by) * p.bs;
    b.ref0 = -1; b.ref1 = -1; b.mv0 = 0; b.mv1 = 0;
    if (uses_list(type, 0)) {
        b.ref0 = (int8_t)r2f[2 + p.i.ref_index[0][4 * (size_t)xy + b8]];
        b.mv0 = reinterpret_cast<const int *>(p.i.motion_val[0])[mvi];
    }
    if (uses_list(type, 1)) {
        b.ref1 = (int8_t)r2f[64 + 2 + p.i.ref_index[1][4 * (size_t)xy + b8]];
        b.mv1 = reinterpret_cast<const int *>(p.i.motion_val[1])[mvi];
    }
    return b;
}

__device__ __forceinline__ int mv_far(int a, int b, int ylim)    // |dx| >= 4 or |dy| >= mvy_limit (4; 2 for the macroblocks of a field, h264_loopfilter.c:723)
{
    const int dx = lo16s(a) - lo16s(b), dy = hi16s(a) - hi16s(b);
    return (abs(dx) >= 4) | (abs(dy) >= ylim);
}

// check_mv(), h264_loopfilter.c:438-469
__device__ __forceinline__ int motion_differs(const Blk &a, const Blk &b, int lists, int ylim)
{
    int v = a.ref0 != b.ref0;
    if (!v && a.ref0 != -1) v = mv_far(a.mv0, b.mv0, ylim);
    if (lists == 2) {
        if (!v) v = (a.ref1 != b.ref1) | mv_far(a.mv1, b.mv1, ylim);
        if (v) {
            if ((a.ref0 != b.ref1) | (a.ref1 != b.ref0)) return 1;
            return mv_far(a.mv0, b.mv1, ylim) | mv_far(a.mv1, b.mv0, ylim);
        }
    }
    return v;
}

struct EdgeOut { uint8_t alpha, beta; int8_t tc[4]; bool intra; };

// filter_mb_edge{v,h,cv,ch}, h264_loopfilter.c:103-236
__device__ __forceinline__ EdgeOut edge_params(const int (&bS)[4], int qp, int offa, int offb, bool may_be_intra, int chroma)
{
    EdgeOut o = { 0, 0, { 0, 0, 0, 0 }, false };
    const int ia = min(qp + offa, 51), ib = min(qp + offb, 51);
    const int alpha = ia < 0 ? 0 : c_alpha[ia], beta = ib < 0 ? 0 : c_beta[ib];
    if (!alpha || !beta) return o;
    o.alpha = (uint8_t)alpha; o.beta = (uint8_t)beta;
    if (bS[0] < 4 || !may_be_intra) {
#pragma unroll
        for (int k = 0; k < 4; k++) o.tc[k] = (int8_t)((bS[k] ? (int)c_tc0[ia][bS[k] - 1] : -1) + chroma);
    } else {
        o.intra = true;
    }
    return o;
}

__global__ void __launch_bounds__(128)
h264_deblock_params_kernel(LfPic p, FFH264DeblockMB *__restrict__ out, int n_mbs)
{
    const int t = blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= 2 * n_mbs) return;
    const int dir = t & 1, m = t >> 1;
    const int per_pic = p.i.mb_w * p.i.mb_h, pic = m / per_pic, mi = m - pic * per_pic;
    const int y = mi / p.i.mb_w, x = mi - y * p.i.mb_w;
    const int row = pic * p.i.mb_h + y, xy = x + row * p.ms;              // pictures are stacked row-wise
    FFH264DeblockMB &rec = out[m];
    // this thread's fields, filled with "edge not filtered"
    uint8_t alpha[4] = { 0, 0, 0, 0 }, beta[4] = { 0, 0, 0, 0 }, intra = 0;
    int8_t tc0[4][4] = {};
    uint8_t calpha[2][2] = {}, cbeta[2][2] = {}, cintra[2] = { 0, 0 };
    int8_t ctc0[2][2][4] = {};
    // chroma_format_idc 2: the four horizontal chroma edges (this thread's when dir == 1) go to the 4:2:2 record
    const bool c422h = p.i.chroma422 != nullptr && dir == 1;
    uint8_t xalpha[2][4] = {}, xbeta[2][4] = {}, xintra[2] = { 0, 0 };
    int8_t xtc0[2][4][4] = {};

    const int sn = p.i.slice_table[xy];
    const FFH264DeblockSlice &sl = p.i.slices[sn];
    const uint32_t type = p.i.mb_type[xy];
    const int qp = p.i.qscale_table[xy];
    bool active = sl.deblocking_filter != 0;
    if (active) {   // low-qp shortcut, h264_slice.c:2085-2107 (the padding entries it reads hold qp 0)
        const int th = sl.qp_thresh;
        const bool has_l = x + y * p.ms - 1 >= 0, has_t = y > 0;
        const int ql = x > 0 ? p.i.qscale_table[xy - 1] : 0, qt = y > 0 ? p.i.qscale_table[xy - p.ms] : 0;
        if (qp <= th && (!has_l || ((qp + ql + 1) >> 1) <= th) && (!has_t || ((qp + qt + 1) >> 1) <= th)) active = false;
    }
    if (active) {
        const int nxy = dir ? xy - p.ms : xy - 1;
        uint32_t mt = (dir ? y > 0 : x > 0) ? p.i.mb_type[nxy] : 0;
        if (mt && sl.deblocking_filter == 2 && p.i.slice_table[nxy] != sn) mt = 0;
        const int offa = sl.alpha_c0_offset, offb = sl.beta_offset, lists = sl.list_count;
        const int mask_edge = dir ? (0x33331130u >> (4 * ((type >> 3) & 7))) & 15 : (0x11113330u >> (4 * ((type >> 3) & 7))) & 15;
        const bool is_intra = type & T_INTRA;
        const int edges = (mask_edge == 3 && !is_intra && !(p.i.cbp_table[xy] & 15)) ? 1 : 4;
        const uint32_t par0 = type & (T_16x16 | (T_8x16 >> dir));
        const int ylim = (type & T_INTERLACED) ? 2 : 4;
        const int cq0 = p.i.chroma_qp_table[qp], cq1 = p.i.chroma_qp_table[64 + qp];
        const int bx4 = 4 * x, by4 = 4 * row, nbx4 = dir ? bx4 : bx4 - 4, nby4 = dir ? by4 - 4 : by4;
        for (int e = 0; e < edges; e++) {
            if (e == 0 && !mt) continue;
            const bool deblock_edge = !(e && (type & T_DCT8) && (e & 1));      // inside an 8x8 transform block there is no luma edge; 4:2:2 chroma still has one (h264_loopfilter.c:633)
            if (!deblock_edge && !c422h) continue;
            int bS[4];
            if (e == 0 && ((type | mt) & T_INTRA)) {
                // 4, but 3 across the horizontal macroblock edges of a field picture (h264_loopfilter.c:551-557)
                bS[0] = bS[1] = bS[2] = bS[3] = (((type | mt) & T_INTERLACED) && !(p.i.field_picture && dir == 0)) ? 3 : 4;
            } else if (is_intra) {
                bS[0] = bS[1] = bS[2] = bS[3] = 3;
            } else {
                int whole = -1;
                if (e && (e & mask_edge)) whole = 0;
                else if (par0 && (e || (mt & (T_16x16 | (T_8x16 >> dir))))) {
                    const Blk a = fetch_block(p, xy, bx4, by4, dir ? 0 : e, dir ? e : 0, type, 0);
                    const Blk b = e ? fetch_block(p, xy, bx4, by4, dir ? 0 : e - 1, dir ? e - 1 : 0, type, 0)
                                    : fetch_block(p, nxy, nbx4, nby4, dir ? 0 : 3, dir ? 3 : 0, mt, dir ? 1 : 2);
                    whole = motion_differs(a, b, lists, ylim);
                }
#pragma unroll
                for (int k = 0; k < 4; k++) {
                    const Blk a = fetch_block(p, xy, bx4, by4, dir ? k : e, dir ? e : k, type, 0);
                    const Blk b = e ? fetch_block(p, xy, bx4, by4, dir ? k : e - 1, dir ? e - 1 : k, type, 0)
                                    : fetch_block(p, nxy, nbx4, nby4, dir ? k : 3, dir ? 3 : k, mt, dir ? 1 : 2);
                    bS[k] = (a.nz | b.nz) ? 2 : whole >= 0 ? whole : motion_differs(a, b, lists, ylim);
                }
            }
            if (!(bS[0] + bS[1] + bS[2] + bS[3])) continue;
            int ql = qp, qc0 = cq0, qc1 = cq1;
            if (e == 0) {
                const int qn = p.i.qscale_table[nxy];
                ql = (qp + qn + 1) >> 1;
                qc0 = (cq0 + p.i.chroma_qp_table[qn] + 1) >> 1;
                qc1 = (cq1 + p.i.chroma_qp_table[64 + qn] + 1) >> 1;
            }
            if (deblock_edge) {
                const EdgeOut L = edge_params(bS, ql, offa, offb, e == 0, 0);
                alpha[e] = L.alpha; beta[e] = L.beta; intra |= (uint8_t)L.intra << e;
#pragma unroll
                for (int k = 0; k < 4; k++) tc0[e][k] = L.tc[k];
            }
            if (c422h) {
                const EdgeOut C0 = edge_params(bS, qc0, offa, offb, e == 0, 1), C1 = edge_params(bS, qc1, offa, offb, e == 0, 1);
                xalpha[0][e] = C0.alpha; xbeta[0][e] = C0.beta; xintra[0] |= (uint8_t)C0.intra << e;
                xalpha[1][e] = C1.alpha; xbeta[1][e] = C1.beta; xintra[1] |= (uint8_t)C1.intra << e;
#pragma unroll
                for (int k = 0; k < 4; k++) { xtc0[0][e][k] = C0.tc[k]; xtc0[1][e][k] = C1.tc[k]; }
            } else if (!(e & 1)) {
                const EdgeOut C0 = edge_params(bS, qc0, offa, offb, e == 0, 1), C1 = edge_params(bS, qc1, offa, offb, e == 0, 1);
                const int ce = e >> 1;
                calpha[0][ce] = C0.alpha; cbeta[0][ce] = C0.beta; cintra[0] |= (uint8_t)C0.intra << ce;
                calpha[1][ce] = C1.alpha; cbeta[1][ce] = C1.beta; cintra[1] |= (uint8_t)C1.intra << ce;
#pragma unroll
                for (int k = 0; k < 4; k++) { ctc0[0][ce][k] = C0.tc[k]; ctc0[1][ce][k] = C1.tc[k]; }
            }
        }
    }
#pragma unroll
    for (int e = 0; e < 4; e++) {
        rec.alpha[dir][e] = alpha[e]; rec.beta[dir][e] = beta[e];
#pragma unroll
        for (int k = 0; k < 4; k++) rec.tc0[dir][e][k] = tc0[e][k];
    }
    rec.intra[dir] = intra;
#pragma unroll
    for (int pl = 0; pl < 2; pl++) {
        rec.cintra[pl][dir] = cintra[pl];
#pragma unroll
        for (int ce = 0; ce < 2; ce++) {
            rec.calpha[pl][dir][ce] = calpha[pl][ce]; rec.cbeta[pl][dir][ce] = cbeta[pl][ce];
#pragma unroll
            for (int k = 0; k < 4; k++) rec.ctc0[pl][dir][ce][k] = ctc0[pl][ce][k];
        }
    }
    rec.pad[dir] = 0;
    if (c422h) {
        FFH264DeblockChroma422 &x = p.i.chroma422[m];
#pragma unroll
        for (int pl = 0; pl < 2; pl++) {
            x.intra[pl] = xintra[pl]; x.pad[pl] = 0;
#pragma unroll
            for (int e = 0; e < 4; e++) {
                x.alpha[pl][e] = xalpha[pl][e]; x.beta[pl][e] = xbeta[pl][e];
#pragma unroll
                for (int k = 0; k < 4; k++) x.tc0[pl][e][k] = xtc0[pl][e][k];
            }
        }
    }
}

}  // namespace avb

using namespace avb;

extern "C" int ff_h264_deblock_params_cuda(const FFH264DeblockInfo *info, FFH264DeblockMB *out, void *stream)
{
    avb::enter();
    if (!info || !out || info->mb_w <= 0 || info->mb_h <= 0 || info->n_pictures <= 0 || info->n_slices <= 0 || info->n_slices > 32) {
        set_error_msg("ff_h264_deblock_params_cuda", "bad arguments (1..32 slices per call: the reference keeps 32 ref2frm tables)");
        return -1;
    }
    LfPic p; p.i = *info; p.ms = info->mb_w + 1; p.bs = 4 * info->mb_w;
    const int n = info->mb_w * info->mb_h * info->n_pictures;
    h264_deblock_params_kernel<<<(2 * n + 127) / 128, 128, 0, (cudaStream_t)stream>>>(p, out, n);
    return check_launch("ff_h264_deblock_params_cuda");
}

// The decoder back-end's flush point (SURVEY 8f rank 1): everything the CPU recorded for a batch of pictures / slices, run in the
// order hl_decode_mb() (libavcodec/h264_mb_template.c:40-260) and loop_filter() (h264_slice.c:1972-2066) impose.  Pure stream
// ordering of the batch entry points -- no host synchronisation; an error of any stage stops the flush.
extern "C" int ff_h264_flush_pictures_cuda(const FFH264PictureWork *w, void *stream)
{
    avb::enter();
    if (!w || w->mb_w <= 0 || w->mb_h <= 0 || w->n_pictures <= 0 || !w->luma || !w->cb || !w->cr) {
        set_error_msg("ff_h264_flush_pictures_cuda", "bad arguments"); return -1;
    }
    const size_t n_mb = (size_t)w->mb_w * w->mb_h * w->n_pictures;
    const int depth = w->bit_depth ? w->bit_depth : 8, idc = w->chroma_format_idc ? w->chroma_format_idc : 1;
    if (depth != 8 || idc != 1) {
        // 9 / 10-bit pictures and / or 4:2:2 chroma: the same order through the kernels of h264_hbd_batch.cu (coeffs / luma_dc hold int32 at 9 / 10 bit)
        if ((depth != 8 && depth != 9 && depth != 10) || (idc != 1 && idc != 2)) { set_error_msg("ff_h264_flush_pictures_cuda", "bit_depth 8 / 9 / 10, chroma_format_idc 1 / 2"); return -1; }
        if (w->n_mc && ff_h264_mc_batch_hbd_cuda(depth, idc, w->mc, w->n_mc, w->refs, w->luma, w->cb, w->cr, w->linesize, w->uvlinesize, 16 * w->mb_w, 16 * w->mb_h, stream)) return -1;
        for (int pl = 0; pl < 3; pl++) {
            uint8_t *plane = pl == 0 ? w->luma : pl == 1 ? w->cb : w->cr;
            if (!w->n_weight[pl]) continue;
            if (depth == 8 ? ff_h264_weight_batch_cuda(w->weight[pl], w->n_weight[pl], plane, w->weight_src[pl], pl ? w->uvlinesize : w->linesize, stream)
                           : ff_h264_weight_batch_hbd_cuda(depth, w->weight[pl], w->n_weight[pl], plane, w->weight_src[pl], pl ? w->uvlinesize : w->linesize, stream)) return -1;
        }
        // (8-bit 4:2:2: int16 coefficients behind w->coeffs / w->luma_dc, as the header says)
        if (w->dc && (depth == 8 ? ff_h264_dc_dequant_batch_422_cuda(w->dc, n_mb, w->coeffs, w->coeff_stride, w->luma_dc, stream)
                                 : ff_h264_dc_dequant_batch_hbd_cuda(idc, w->dc, n_mb, (int32_t *)w->coeffs, w->coeff_stride, (const int32_t *)w->luma_dc, stream))) return -1;
        if (w->residual && ff_h264_idct_add_mb_batch_hbd_cuda(depth, idc, w->residual, n_mb, (int32_t *)w->coeffs, w->coeff_stride, w->nnzc, w->luma, w->cb, w->cr,
                                                              w->linesize, w->uvlinesize, stream)) return -1;
        if (w->intra && (idc == 2 ? ff_h264_intra_mb_batch_422_cuda(depth, w->intra, w->mb_w, w->mb_h, w->n_pictures, w->coeffs, w->coeff_stride, w->nnzc, w->luma, w->cb, w->cr,
                                                                    w->linesize, w->uvlinesize, stream)
                                  : ff_h264_intra_mb_batch_hbd_cuda(depth, w->intra, w->mb_w, w->mb_h, w->n_pictures, (int32_t *)w->coeffs, w->coeff_stride, w->nnzc, w->luma, w->cb, w->cr,
                                                                    w->linesize, w->uvlinesize, stream))) return -1;
        if (w->deblock_info) {
            if (!w->deblock_records || w->deblock_info->mb_w != w->mb_w || w->deblock_info->mb_h != w->mb_h || w->deblock_info->n_pictures != w->n_pictures ||
                (idc == 2) != (w->deblock_info->chroma422 != nullptr)) {
                set_error_msg("ff_h264_flush_pictures_cuda", "deblock_info does not describe this batch"); return -1;
            }
            if (ff_h264_deblock_params_cuda(w->deblock_info, w->deblock_records, stream)) return -1;
        }
        if (w->deblock_records) {
            if (idc == 2) {
                const FFH264DeblockChroma422 *x = w->deblock_info ? w->deblock_info->chroma422 : w->deblock_chroma422;
                if (ff_h264_deblock_batch_422_cuda(depth, w->deblock_records, x, w->mb_w, w->mb_h, w->n_pictures, w->luma, w->cb, w->cr, w->linesize, w->uvlinesize, stream)) return -1;
            } else if (ff_h264_deblock_batch_hbd_cuda(depth, w->deblock_records, w->mb_w, w->mb_h, w->n_pictures, w->luma, w->cb, w->cr, w->linesize, w->uvlinesize, stream)) return -1;
        }
        return 0;
    }
    // an intra arena stage 5 would refuse is refused before stage 1 writes anything
    if (w->intra && !h264_intra_args_ok("ff_h264_flush_pictures_cuda", w->intra, w->coeffs, w->coeff_stride, w->nnzc, w->luma, w->cb, w->cr,
                                        w->linesize, w->uvlinesize, w->progress)) return -1;
    // 1. inter prediction: every put partition, then every avg partition (h264_mb.c:322-366)
    if (w->n_mc && ff_h264_mc_batch_cuda(w->mc, w->n_mc, w->refs, w->luma, w->cb, w->cr, w->linesize, w->uvlinesize, 16 * w->mb_w, 16 * w->mb_h, stream)) return -1;
    // 2. explicit / implicit weighted prediction on the predicted blocks (h264_mb.c:368-460), plane by plane
    for (int pl = 0; pl < 3; pl++) {
        uint8_t *plane = pl == 0 ? w->luma : pl == 1 ? w->cb : w->cr;
        if (w->n_weight[pl] && ff_h264_weight_batch_cuda(w->weight[pl], w->n_weight[pl], plane, w->weight_src[pl], pl ? w->uvlinesize : w->linesize, stream)) return -1;
    }
    // 3. DC transforms + dequantisation into the coefficient arena, 4. residual of the inter macroblocks
    if (w->dc && ff_h264_dc_dequant_batch_cuda(w->dc, n_mb, w->coeffs, w->coeff_stride, w->luma_dc, stream)) return -1;
    if (w->residual && ff_h264_idct_add_mb_batch_cuda(w->residual, n_mb, w->coeffs, w->coeff_stride, w->nnzc, w->luma, w->cb, w->cr, w->linesize, w->uvlinesize, stream)) return -1;
    // 5. intra macroblocks: prediction interleaved with their residual, as a wavefront over the reconstructed neighbours
    if (w->intra && ff_h264_intra_mb_batch_cuda(w->intra, w->mb_w, w->mb_h, w->n_pictures, w->coeffs, w->coeff_stride, w->nnzc, w->luma, w->cb, w->cr,
                                                w->linesize, w->uvlinesize, w->progress, stream)) return -1;
    // 6. deblocking decisions from the side information, 7. the loop filter
    if (w->deblock_info) {
        if (!w->deblock_records || w->deblock_info->mb_w != w->mb_w || w->deblock_info->mb_h != w->mb_h || w->deblock_info->n_pictures != w->n_pictures) {
            set_error_msg("ff_h264_flush_pictures_cuda", "deblock_info does not describe this batch"); return -1;
        }
        if (ff_h264_deblock_params_cuda(w->deblock_info, w->deblock_records, stream)) return -1;
    }
    if (w->deblock_records && ff_h264_deblock_batch_cuda(w->deblock_records, w->mb_w, w->mb_h, w->n_pictures, w->luma, w->cb, w->cr, w->linesize, w->uvlinesize,
                                                         w->progress, stream)) return -1;
    return 0;
}
