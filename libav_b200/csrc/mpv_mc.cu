// libav_b200/csrc/mpv_mc.cu -- batched mpegvideo motion compensation (ff_mpv_motion, libavcodec/mpegvideo_motion.c) and the picture flush
// point of an MPEG-1 / MPEG-2 / H.263 / MPEG-4 decoder back-end.
//
// One warp per macroblock record, one lane per destination column (mpv_mc_block.cuh; OBMC pictures and S-VOPs in kernels of their own,
// mpv_obmc.cuh and mpv_gmc.cuh; MPEG-2 4:2:2 and 4:4:4 pictures and interlaced MPEG-4 pictures in instances of the same body that run in
// launches of their own, so progressive 4:2:0 pictures run the code they ran before).  Up to MPV_PICS_PER_LAUNCH pictures travel as
// kernel parameters; a warp finds its picture by scanning their record offsets.  The pictures' checks are all made on the host before
// anything is launched, so a refused call leaves the destination as it was.
#include "mpv_mc_block.cuh"
#include "mpv_obmc.cuh"
#include "mpv_gmc.cuh"
#include "h263_lf.cuh"
#include <algorithm>

namespace avb {

enum { MPV_PICS_PER_LAUNCH = 16 };

struct MpvMcLaunch {
    MpvMcPic pic[MPV_PICS_PER_LAUNCH];
    const FFMpvMCRecord *recs[MPV_PICS_PER_LAUNCH];
    unsigned long long start[MPV_PICS_PER_LAUNCH + 1];     // first warp of each picture; start[n] = warps in the launch
    int n;
    uint32_t *rejected;
};

// the warp's record of a launch, the picture kind's body on it (CF, IL: mpv_mc_block.cuh)
template <int CF, int IL>
__device__ __forceinline__ void mpv_mc_warp(const MpvMcLaunch &L)
{
    const unsigned long long w = (unsigned long long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    if (w >= L.start[L.n]) return;
    int p = 0;
    while (p + 1 < L.n && w >= L.start[p + 1]) p++;
    const MpvMcPic &P = L.pic[p];
    const FFMpvMCRecord r = L.recs[p][w - L.start[p]];
    if (mpv_mc_reject_kind<IL>(P, r)) {
        if ((threadIdx.x & 31) == 0) atomicAdd(L.rejected, 1u);
        return;
    }
    mpv_mc_lane<CF, IL>(P, r, threadIdx.x & 31);
}

__global__ void __launch_bounds__(128) mpv_mc_kernel(const __grid_constant__ MpvMcLaunch L) { mpv_mc_warp<1, 0>(L); }

// MPEG-2 4:2:2 (CF 2) and 4:4:4 (CF 3) pictures
template <int CF>
__global__ void __launch_bounds__(128) mpv_mc_chroma_kernel(const __grid_constant__ MpvMcLaunch L) { mpv_mc_warp<CF, 0>(L); }

// interlaced MPEG-4 pictures (interlaced set in out_format 2) other than S-VOPs
__global__ void __launch_bounds__(128) mpv_mc_ilace_kernel(const __grid_constant__ MpvMcLaunch L) { mpv_mc_warp<1, 1>(L); }

// OBMC pictures (obmc set in a P picture): the same walk, with each record's FFMpvOBMCRecord and put_obmc's weights
struct MpvObmcLaunch {
    MpvMcPic pic[MPV_PICS_PER_LAUNCH];
    const FFMpvMCRecord *recs[MPV_PICS_PER_LAUNCH];
    const FFMpvOBMCRecord *obmc[MPV_PICS_PER_LAUNCH];
    unsigned long long start[MPV_PICS_PER_LAUNCH + 1];
    int n;
    uint32_t *rejected;
    uint8_t weights[64];
};

__global__ void __launch_bounds__(128) mpv_obmc_kernel(const __grid_constant__ MpvObmcLaunch L)
{
    const unsigned long long w = (unsigned long long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    if (w >= L.start[L.n]) return;
    int p = 0;
    while (p + 1 < L.n && w >= L.start[p + 1]) p++;
    const MpvMcPic &P = L.pic[p];
    const FFMpvMCRecord r = L.recs[p][w - L.start[p]];
    if (mpv_obmc_reject(P, r)) {
        if ((threadIdx.x & 31) == 0) atomicAdd(L.rejected, 1u);
        return;
    }
    const FFMpvOBMCRecord o = L.obmc[p][w - L.start[p]];
    mpv_obmc_lane(P, r, o, L.weights, threadIdx.x & 31);
}

// S-VOPs (sprite set): the same walk, with each picture's sprite parameters and the records' mcsel
struct MpvGmcLaunch {
    MpvMcPic pic[MPV_PICS_PER_LAUNCH];
    MpvGmcParams gmc[MPV_PICS_PER_LAUNCH];
    const FFMpvMCRecord *recs[MPV_PICS_PER_LAUNCH];
    unsigned long long start[MPV_PICS_PER_LAUNCH + 1];
    int n;
    uint32_t *rejected;
};

template <int IL>
__device__ __forceinline__ void mpv_gmc_warp(const MpvGmcLaunch &L)
{
    const unsigned long long w = (unsigned long long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    if (w >= L.start[L.n]) return;
    int p = 0;
    while (p + 1 < L.n && w >= L.start[p + 1]) p++;
    const MpvMcPic &P = L.pic[p];
    const FFMpvMCRecord r = L.recs[p][w - L.start[p]];
    if (mpv_mc_reject_kind<IL>(P, r)) {
        if ((threadIdx.x & 31) == 0) atomicAdd(L.rejected, 1u);
        return;
    }
    mpv_gmc_lane<IL>(P, L.gmc[p], r, threadIdx.x & 31);
}

__global__ void __launch_bounds__(128) mpv_gmc_kernel(const __grid_constant__ MpvGmcLaunch L) { mpv_gmc_warp<0>(L); }

// interlaced S-VOPs: their non-mcsel records may be FIELD ones
__global__ void __launch_bounds__(128) mpv_gmc_ilace_kernel(const __grid_constant__ MpvGmcLaunch L) { mpv_gmc_warp<1>(L); }

namespace {

int refuse(const char *msg) { set_error_msg("ff_mpv_motion_batch_cuda", msg); return -1; }

// the frame the picture writes: dest[0] of a bottom field starts one line into it
const uint8_t *frame_base(const FFMpvMCPicture &q) { return q.dest[0] - (q.picture_structure == 2 ? q.linesize : 0); }

// apply_obmc runs instead of ff_mpv_motion (mpegvideo_motion.c:829-831)
bool mpv_obmc_picture(const FFMpvMCPicture &q) { return q.obmc && !q.b_picture; }

// the kernel a picture goes to, in launch order (an accepted sprite picture is never an OBMC one, an accepted OBMC picture never
// interlaced, and chroma other than 4:2:0 is MPEG-1 / MPEG-2's alone)
enum { MPV_K_PLAIN, MPV_K_OBMC, MPV_K_GMC, MPV_K_422, MPV_K_444, MPV_K_ILACE, MPV_K_GMC_ILACE, MPV_KINDS };

int mpv_kernel_of(const FFMpvMCPicture &q)
{
    const bool il = q.out_format == 2 && q.interlaced;
    if (q.sprite) return il ? MPV_K_GMC_ILACE : MPV_K_GMC;
    if (mpv_obmc_picture(q)) return MPV_K_OBMC;
    if (q.chroma_format != 1) return q.chroma_format == 2 ? MPV_K_422 : MPV_K_444;
    return il ? MPV_K_ILACE : MPV_K_PLAIN;
}

MpvGmcParams mpv_gmc_params(const FFMpvMCPicture &q)
{
    MpvGmcParams G;
    G.acc = q.sprite_warping_accuracy;
    G.pts = q.real_sprite_warping_points;
    memcpy(G.off, q.sprite_offset, sizeof(G.off));
    memcpy(G.delta, q.sprite_delta, sizeof(G.delta));
    return G;
}

// the picture-level checks; fills the kernel's view of the picture
int mpv_picture(const FFMpvMCPicture &q, MpvMcPic &P)
{
    if (q.out_format == 1) return refuse("H.261 is not supported");
    if (q.out_format != 0 && q.out_format != 2) return refuse("out_format must be 0 (MPEG-1 / MPEG-2) or 2 (H.263 / MPEG-4)");
    if (q.obmc && !q.b_picture && (q.out_format != 2 || q.quarter_sample || (q.n_recs && !q.obmc_recs)))
        return refuse("OBMC is supported in half-sample H.263-family P pictures with obmc_recs only");
    if (q.sprite && (q.out_format != 2 || q.picture_structure != 3 || q.b_picture || q.obmc || q.real_sprite_warping_points < 1 ||
                     q.real_sprite_warping_points > 3 || q.sprite_warping_accuracy < 0 || q.sprite_warping_accuracy > 3))
        return refuse("GMC / sprite pictures are supported as MPEG-4 frame S-VOPs without OBMC, with real_sprite_warping_points 1..3 "
                      "and sprite_warping_accuracy 0..3 only");
    if (q.mspel) return refuse("WMV2 mspel is not supported");
    if (q.lowres) return refuse("lowres is not supported");
    if (q.chroma_format < 1 || q.chroma_format > 3 || (q.chroma_format != 1 && q.out_format != 0))
        return refuse("chroma_format must be 1 (4:2:0), or 2 (4:2:2) / 3 (4:4:4) in MPEG-1 / MPEG-2 pictures");
    if (q.out_format == 2 && q.interlaced && q.obmc && !q.b_picture) return refuse("OBMC is not supported in interlaced P pictures");
    if (q.picture_structure < 1 || q.picture_structure > 3) return refuse("picture_structure must be 1, 2 or 3");
    const bool frame = q.picture_structure == 3, h263 = q.out_format == 2;
    if (h263 && !frame) return refuse("field pictures are not supported in the H.263 family");
    if (q.mb_width <= 0 || q.mb_height <= 0 || q.mb_width > 4096 || q.mb_height > 4096 || (!frame && (q.mb_height & 1)))
        return refuse("bad macroblock dimensions");
    const int cx = q.chroma_format != 3, cy = q.chroma_format == 1;    // chroma_x_shift, chroma_y_shift
    if (q.linesize < 16 * q.mb_width + 1 || q.uvlinesize < (16 >> cx) * q.mb_width + 1 || (q.linesize | q.uvlinesize) < 0)
        return refuse("linesize / uvlinesize must exceed the macroblock-aligned width of the plane");
    const int k = frame ? 1 : 2;
    if (q.pic_linesize != k * q.linesize || q.pic_uvlinesize != k * q.uvlinesize)
        return refuse("pic_linesize must be linesize (frame pictures) or 2 * linesize (field pictures)");
    if (q.width <= 0 || q.height <= 0 || q.width > 16 * q.mb_width || q.height > 16 * q.mb_height)
        return refuse("width / height outside the macroblock-aligned picture");
    const int v_max = frame ? 16 * q.mb_height : 8 * q.mb_height;
    if (q.h_edge_pos < 2 || q.v_edge_pos < 2 || q.h_edge_pos > 16 * q.mb_width || q.v_edge_pos > v_max)
        return refuse("h_edge_pos / v_edge_pos outside the macroblock-aligned picture");
    if (!q.dest[0] || !q.dest[1] || !q.dest[2]) return refuse("NULL destination plane");
    if (!frame && !q.first_field && (!q.cur[0] || !q.cur[1] || !q.cur[2]))
        return refuse("a second field needs cur, the planes of its own frame");
    if (q.n_recs && !q.recs) return refuse("NULL record array");
    if (q.cur[0] && q.cur[0] != frame_base(q)) return refuse("cur must be the frame that dest belongs to");
    if (q.last[0] == frame_base(q) || q.next[0] == frame_base(q)) return refuse("last / next is the picture being reconstructed");
    P = MpvMcPic();
    for (int i = 0; i < 3; i++) { P.dest[i] = q.dest[i]; P.cur[i] = q.cur[i]; P.ref[0][i] = q.last[i]; P.ref[1][i] = q.next[i]; }
    P.ls[0] = q.linesize; P.ls[1] = q.uvlinesize; P.pic_k = k;
    P.mb_w = q.mb_width; P.mb_rows = frame ? q.mb_height : q.mb_height >> 1;
    P.width = q.width; P.height = q.height; P.h_edge = q.h_edge_pos; P.v_edge = q.v_edge_pos;
    P.h263 = h263; P.structure = q.picture_structure; P.first_field = q.first_field != 0; P.b_pic = q.b_picture != 0;
    P.no_rnd = q.no_rounding != 0; P.bugs = q.workaround_bugs; P.qpel = h263 && q.quarter_sample;
    P.rw[0] = 16 * q.mb_width + 1; P.rh[0] = 16 * q.mb_height + 1;
    P.rw[1] = (16 >> cx) * q.mb_width + 1; P.rh[1] = (16 >> cy) * q.mb_height + 1;
    return 0;
}

// the pictures, records and warp starts of one launch of the pictures pics[idx[0..m)]; returns the launch's warps
template <class Launch>
unsigned long long mpv_fill(Launch &L, const FFMpvMCPicture *pics, const MpvMcPic *P, const int *idx, int m, uint32_t *rejected)
{
    memset(&L, 0, sizeof(L));
    L.n = m;
    L.rejected = rejected;
    for (int p = 0; p < m; p++) {
        L.pic[p] = P[idx[p]];
        L.recs[p] = pics[idx[p]].recs;
        L.start[p + 1] = L.start[p] + pics[idx[p]].n_recs;
    }
    return L.start[m];
}

// one launch of kind k (mpv_kernel_of) over the pictures pics[idx[0..m)], m <= MPV_PICS_PER_LAUNCH
int mpv_launch(int k, const FFMpvMCPicture *pics, const MpvMcPic *P, const int *idx, int m, uint32_t *rejected, cudaStream_t stream)
{
    if (k == MPV_K_OBMC) {
        MpvObmcLaunch L;
        const unsigned long long warps = mpv_fill(L, pics, P, idx, m, rejected);
        if (!warps) return 0;
        memcpy(L.weights, mpv_obmc_weights, sizeof(L.weights));
        for (int p = 0; p < m; p++) L.obmc[p] = pics[idx[p]].obmc_recs;
        AVB_LAUNCH(mpv_obmc_kernel, (unsigned)((warps + 3) / 4), 128, 0, stream)(L);
    } else if (k == MPV_K_GMC || k == MPV_K_GMC_ILACE) {
        MpvGmcLaunch L;
        const unsigned long long warps = mpv_fill(L, pics, P, idx, m, rejected);
        if (!warps) return 0;
        for (int p = 0; p < m; p++) L.gmc[p] = mpv_gmc_params(pics[idx[p]]);
        if (k == MPV_K_GMC) AVB_LAUNCH(mpv_gmc_kernel, (unsigned)((warps + 3) / 4), 128, 0, stream)(L);
        else                AVB_LAUNCH(mpv_gmc_ilace_kernel, (unsigned)((warps + 3) / 4), 128, 0, stream)(L);
    } else {
        MpvMcLaunch L;
        const unsigned long long warps = mpv_fill(L, pics, P, idx, m, rejected);
        if (!warps) return 0;
        const unsigned grid = (unsigned)((warps + 3) / 4);
        if (k == MPV_K_PLAIN)      AVB_LAUNCH(mpv_mc_kernel, grid, 128, 0, stream)(L);
        else if (k == MPV_K_422)   AVB_LAUNCH(mpv_mc_chroma_kernel<2>, grid, 128, 0, stream)(L);
        else if (k == MPV_K_444)   AVB_LAUNCH(mpv_mc_chroma_kernel<3>, grid, 128, 0, stream)(L);
        else                       AVB_LAUNCH(mpv_mc_ilace_kernel, grid, 128, 0, stream)(L);
    }
    return check_launch("ff_mpv_motion_batch_cuda");
}

}  // namespace

}  // namespace avb

using namespace avb;

extern "C" int ff_mpv_motion_batch_cuda(const FFMpvMCPicture *pics, int n, uint32_t *rejected, void *stream)
{
    if (n == 0) return 0;
    if (!pics || n < 0 || !rejected) return refuse("NULL pictures / rejected counter, or a negative count");
    MpvMcPic *P = new MpvMcPic[n];
    int rc = 0;
    for (int i = 0; i < n && !rc; i++) rc = mpv_picture(pics[i], P[i]);
    // by frame base: two fields of one frame, or a picture whose frame another one predicts from, cannot share a call
    for (int i = 0; i < n && !rc; i++)
        for (int j = 0; j < n && !rc; j++) {
            const uint8_t *b = frame_base(pics[i]);
            if (i != j && (b == frame_base(pics[j]) || b == pics[j].last[0] || b == pics[j].next[0]))
                rc = refuse("pictures of one call write the same frame or read each other (a second field predicting from its first field, "
                            "or a picture predicting from another of the call, goes into a later call)");
        }
    if (!rc) {
        enter();
        // each kind of picture in launches of its own, in mpv_kernel_of's order; pictures of a call are independent
        int *order = new int[n], first[MPV_KINDS + 1] = {};
        for (int k = 0, m = 0; k < MPV_KINDS; k++) {
            first[k] = m;
            for (int i = 0; i < n; i++)
                if (mpv_kernel_of(pics[i]) == k) order[m++] = i;
            first[k + 1] = m;
        }
        for (int k = 0; k < MPV_KINDS && !rc; k++)
            for (int g = first[k]; g < first[k + 1] && !rc; g += MPV_PICS_PER_LAUNCH)
                rc = mpv_launch(k, pics, P, order + g, std::min(first[k + 1] - g, (int)MPV_PICS_PER_LAUNCH), rejected, (cudaStream_t)stream);
        delete[] order;
    }
    delete[] P;
    return rc;
}

// ---- the H.263 loop filter over whole pictures (h263_lf.cuh)

namespace avb {
namespace {

int lf_refuse(const char *msg) { set_error_msg("ff_h263_loop_filter_batch_cuda", msg); return -1; }

// the picture-level checks; fills the kernel's view of the picture
int h263_lf_picture(const FFH263LoopFilterPicture &q, H263LfPic &P)
{
    if (q.mb_width <= 0 || q.mb_height <= 0 || q.mb_width > 4096 || q.mb_height > 4096) return lf_refuse("bad macroblock dimensions");
    if (q.mb_stride <= q.mb_width) return lf_refuse("mb_stride must exceed mb_width");
    if (q.linesize < 16 * q.mb_width || q.uvlinesize < 8 * q.mb_width) return lf_refuse("linesize / uvlinesize below the macroblock-aligned width");
    if (!q.data[0] || !q.data[1] || !q.data[2] || !q.mb_type || !q.qscale_table) return lf_refuse("NULL plane or table");
    for (int i = 0; i < 32; i++)
        if (q.chroma_qscale_table[i] > 31) return lf_refuse("chroma_qscale_table entries must be 0..31");
    P = H263LfPic();
    for (int i = 0; i < 3; i++) P.data[i] = q.data[i];
    P.ls[0] = q.linesize; P.ls[1] = q.uvlinesize;
    P.mb_w = q.mb_width; P.mb_h = q.mb_height; P.mb_stride = q.mb_stride;
    P.mb_type = q.mb_type; P.qscale = q.qscale_table;
    for (int i = 0; i < 32; i++) {
        P.strength[0][i] = h263_lf_strength_tab[i];
        P.strength[1][i] = h263_lf_strength_tab[q.chroma_qscale_table[i]];
    }
    return 0;
}

// the bytes plane pl of a picture spans (its last row ends at the aligned width)
void h263_lf_span(const FFH263LoopFilterPicture &q, int pl, uintptr_t &lo, uintptr_t &hi)
{
    const int c = pl != 0;
    lo = (uintptr_t)q.data[pl];
    hi = lo + (uintptr_t)((16 >> c) * q.mb_height - 1) * (uintptr_t)(c ? q.uvlinesize : q.linesize) + (uintptr_t)((16 >> c) * q.mb_width);
}

// every check of a call, made before anything is launched
int h263_lf_check(const FFH263LoopFilterPicture *pics, int n, H263LfPic *P)
{
    if (!pics || n < 0) return lf_refuse("NULL pictures or a negative count");
    for (int i = 0; i < n; i++)
        if (h263_lf_picture(pics[i], P[i])) return -1;
    // the planes' spans by start address: a span that begins before the furthest end seen so far overlaps the span reaching that end,
    // and the first overlap between two pictures in this order is always one of those
    struct Span { uintptr_t lo, hi; int pic; };
    Span *sp = new Span[3 * (size_t)n];
    for (int i = 0; i < n; i++)
        for (int pl = 0; pl < 3; pl++) { sp[3 * i + pl].pic = i; h263_lf_span(pics[i], pl, sp[3 * i + pl].lo, sp[3 * i + pl].hi); }
    std::sort(sp, sp + 3 * (size_t)n, [](const Span &a, const Span &b) { return a.lo < b.lo; });
    int rc = 0;
    uintptr_t end = 0;
    int end_pic = -1;
    for (size_t k = 0; k < 3 * (size_t)n && !rc; k++) {
        if (sp[k].lo < end && sp[k].pic != end_pic) rc = lf_refuse("two pictures of one call share a frame");
        if (sp[k].hi > end) { end = sp[k].hi; end_pic = sp[k].pic; }
    }
    delete[] sp;
    return rc;
}

int h263_lf_run(const FFH263LoopFilterPicture *pics, const H263LfPic *P, int n, cudaStream_t stream)
{
    for (int g = 0; g < n; g += H263_LF_PICS_PER_LAUNCH) {
        const int m = n - g < H263_LF_PICS_PER_LAUNCH ? n - g : H263_LF_PICS_PER_LAUNCH;
        H263LfLaunch L;
        memset(&L, 0, sizeof(L));
        unsigned most = 0;
        for (int p = 0; p < m; p++) {
            L.pic[p] = P[g + p];
            const unsigned t = (unsigned)(2 * pics[g + p].mb_height + 1) * (unsigned)(2 * pics[g + p].mb_width + 1);     // luma tiles
            most = t > most ? t : most;
        }
        AVB_LAUNCH(h263_lf_kernel, dim3((most + 127) / 128, 3 * m), 128, 0, stream)(L);
        if (check_launch("ff_h263_loop_filter_batch_cuda")) return -1;
    }
    return 0;
}

}  // namespace
}  // namespace avb

extern "C" int ff_h263_loop_filter_batch_cuda(const FFH263LoopFilterPicture *pics, int n, void *stream)
{
    using namespace avb;
    if (n == 0) return 0;
    H263LfPic *P = new H263LfPic[n > 0 ? n : 1];
    int rc = h263_lf_check(pics, n, P);
    if (!rc) {
        enter();
        rc = h263_lf_run(pics, P, n, (cudaStream_t)stream);
    }
    delete[] P;
    return rc;
}

// the stages of a flush, every check but the motion compensation's (made by its own call, the first stage) already passed
static int mpv_flush_run(const FFMpvPictureWork *w, const H263LfPic *lf, void *stream)
{
    if (w->n_pictures && ff_mpv_motion_batch_cuda(w->pictures, w->n_pictures, w->rejected, stream)) return -1;
    for (int i = 0; i < w->n_residual; i++) {
        const FFMpvResidualBatch &b = w->residual[i];
        if (!b.n) continue;
        int rc;
        if (b.dequant < 0)
            rc = b.transform == 3 ? ff_faanidct_batch_cuda(b.mode, b.blocks, b.frame, b.dst_off, b.stride, b.n, 0, b.clear, stream)
               : b.transform      ? ff_xvid_idct_batch_cuda(b.mode, b.blocks, b.frame, b.dst_off, b.stride, b.n, 0, b.clear, stream)
                                  : ff_simple_idct_batch_cuda(b.mode, b.blocks, b.frame, b.dst_off, b.stride, b.n, 0, b.clear, stream);
        else
            rc = b.transform == 3 ? ff_mpeg_dequant_faanidct_batch_cuda(b.dequant, b.tables, b.recs, b.blocks, b.frame, b.dst_off, b.stride, b.n, 0, b.clear, stream)
               : b.transform      ? ff_mpeg_dequant_xvid_idct_batch_cuda(b.dequant, b.tables, b.recs, b.blocks, b.frame, b.dst_off, b.stride, b.n, 0, b.clear, stream)
                                  : ff_mpeg_dequant_idct_batch_cuda(b.dequant, b.tables, b.recs, b.blocks, b.frame, b.dst_off, b.stride, b.n, 0, b.clear, stream);
        if (rc) return -1;
    }
    if (!w->n_loop_filter) return 0;
    enter();
    return h263_lf_run(w->loop_filter, lf, w->n_loop_filter, (cudaStream_t)stream);
}

extern "C" int ff_mpv_flush_pictures_cuda(const FFMpvPictureWork *w, void *stream)
{
    const char *where = "ff_mpv_flush_pictures_cuda";
    if (!w || w->n_pictures < 0 || w->n_residual < 0 || (w->n_residual && !w->residual)) { set_error_msg(where, "bad arguments"); return -1; }
    for (int i = 0; i < w->n_residual; i++) {
        const FFMpvResidualBatch &b = w->residual[i];
        if (b.transform < 0 || b.transform == 2 || b.transform > 3 || b.dequant < -1 || b.dequant > 6 || (b.dequant < 0 && b.mode != 0 && b.mode != 1) ||
            (b.dequant >= 0 && (!b.tables || !b.recs)) || (b.n && (!b.blocks || !b.frame || !b.dst_off))) {
            set_error_msg(where, "bad residual batch: transform 0 / 1 / 3, dequant -1..6, mode 0 / 1, blocks, frame and dst_off set");
            return -1;
        }
    }
    if (w->n_loop_filter < 0 || (w->n_loop_filter && !w->loop_filter)) { set_error_msg(where, "bad loop filter pictures"); return -1; }
    H263LfPic *lf = new H263LfPic[w->n_loop_filter > 0 ? w->n_loop_filter : 1];
    int rc = w->n_loop_filter ? h263_lf_check(w->loop_filter, w->n_loop_filter, lf) : 0;
    if (!rc) rc = mpv_flush_run(w, lf, stream);
    delete[] lf;
    return rc;
}
