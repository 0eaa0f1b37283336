// libav_b200/csrc/mpv_gmc.cuh -- MPEG-4 global motion compensation: gmc1_motion / gmc_motion (libavcodec/mpegvideo_motion.c:37-190) with
// the MpegVideoDSPContext arithmetic they call (gmc1_c, ff_gmc_c: libavcodec/mpegvideodsp.c:24-108), one lane per destination column like
// mpv_mc_block.cuh, whose fetch / store / hpel helpers and plain body it reuses.  A separate kernel (mpv_gmc_kernel in mpv_mc.cu;
// mpv_gmc_ilace_kernel for interlaced ones) runs S-VOPs, so the plain MC kernel is unchanged.  Lanes never communicate: tests/hostsim/ runs
// the body.  The slot kernel of MpegVideoDSPContext (mpegvideodsp.cu) shares the two sample functions.
#pragma once
#include "mpv_mc_block.cuh"

namespace avb {

// the sprite parameters of an S-VOP (FFMpvMCPicture): sprite_warping_accuracy, real_sprite_warping_points, sprite_offset, sprite_delta
struct MpvGmcParams {
    int acc, pts;
    int off[2][2], delta[2][2];
};

// gmc1_c at sample (j, i) of the block whose source starts at t(0, 0): bilinear weights in 1/16 steps, rounder added before >> 8
template <class T>
__device__ __forceinline__ int mpv_gmc1_sample(T t, int j, int i, int x16, int y16, int rounder)
{
    const int A = (16 - x16) * (16 - y16), B = x16 * (16 - y16), C = (16 - x16) * y16, D = x16 * y16;
    return (A * t(j, i) + B * t(j + 1, i) + C * t(j, i + 1) + D * t(j + 1, i + 1) + rounder) >> 8;
}

// ff_gmc_c for the sample whose position is (vx, vy) in 1/65536 units of its 1/(1 << shift) grid: the same four branches, with width /
// height the readable extent of the plane (before the C code's decrement); t(x, y) reads plane sample (x, y), always inside it
template <class T>
__device__ __forceinline__ int mpv_gmc_sample(T t, uint32_t vx, uint32_t vy, int shift, int r, int width, int height)
{
    const int s = 1 << shift;
    int src_x = (int)vx >> 16, src_y = (int)vy >> 16;
    const int frac_x = src_x & (s - 1), frac_y = src_y & (s - 1);
    src_x >>= shift;
    src_y >>= shift;
    width--;
    height--;
    if ((unsigned)src_x < (unsigned)width) {
        if ((unsigned)src_y < (unsigned)height)
            return ((t(src_x, src_y) * (s - frac_x) + t(src_x + 1, src_y) * frac_x) * (s - frac_y) +
                    (t(src_x, src_y + 1) * (s - frac_x) + t(src_x + 1, src_y + 1) * frac_x) * frac_y + r) >> (shift * 2);
        const int y = min(max(src_y, 0), height);
        return ((t(src_x, y) * (s - frac_x) + t(src_x + 1, y) * frac_x) * s + r) >> (shift * 2);
    }
    const int x = min(max(src_x, 0), width);
    if ((unsigned)src_y < (unsigned)height)
        return ((t(x, src_y) * (s - frac_y) + t(x, src_y + 1) * frac_y) * s + r) >> (shift * 2);
    return t(x, min(max(src_y, 0), height));
}

// gmc1_motion: the translation sprite_offset at 1/(2 << acc) sample, as a gmc1_c call on a 17 x 17 luma / 9 x 9 chroma window -- or,
// where the luma fraction is a whole or half sample, the put / put_no_rnd half-sample function
__device__ __forceinline__ void mpv_gmc1_motion(const MpvMcPic &P, const MpvGmcParams &G, const MpvLane &L, const FFMpvMCRecord &r,
                                                const uint8_t *const *ref)
{
    const int c = L.pl != 0, bs = c ? 8 : 16, rounder = 128 - P.no_rnd;
    const int w = P.width >> c, h = P.height >> c, ew = P.h_edge >> c, eh = P.v_edge >> c;
    int mx = G.off[c][0], my = G.off[c][1];
    int src_x = r.mb_x * bs + (mx >> (G.acc + 1)), src_y = r.mb_y * bs + (my >> (G.acc + 1));
    mx = (int)((unsigned)mx << (3 - G.acc));
    my = (int)((unsigned)my << (3 - G.acc));
    src_x = min(max(src_x, -bs), w);                 // the picture's width / height, not h_edge_pos / v_edge_pos
    if (src_x == w) mx = 0;
    src_y = min(max(src_y, -bs), h);
    if (src_y == h) my = 0;
    const int emu = (unsigned)src_x >= (unsigned)max(ew - (bs + 1), 0) || (unsigned)src_y >= (unsigned)max(eh - (bs + 1), 0);
    const MpvSrc s = { ref[L.pl], src_x, src_y, 1, 0, emu, ew, eh };
    if (!c && !((mx | my) & 7)) {
        mpv_hpel(P, L, 0, 0, 16, 0, 1, 16, s, ((mx >> 3) & 1) | ((my >> 2) & 2), P.no_rnd, 0);
        return;
    }
    const auto t = [&](int x, int y) { return mpv_fetch(P, L.pl, s, x, y); };
    for (int i = 0; i < bs; i++) mpv_store(L, i, mpv_gmc1_sample(t, L.c, i, mx & 15, my & 15, rounder), 0);
}

// gmc_motion: the affine map of sprite_offset / sprite_delta through ff_gmc_c.  Sample (x, y) of the block is at ox + dxx * x + dxy * y
// (vy likewise): C's running sums mod 2^32, and the two 8-wide luma calls are one 16-wide map
__device__ __forceinline__ void mpv_gmc_motion(const MpvMcPic &P, const MpvGmcParams &G, const MpvLane &L, const FFMpvMCRecord &r,
                                               const uint8_t *const *ref)
{
    const int c = L.pl != 0, bs = c ? 8 : 16;
    const uint32_t dxx = G.delta[0][0], dxy = G.delta[0][1], dyx = G.delta[1][0], dyy = G.delta[1][1];
    const uint32_t mbx = (uint32_t)r.mb_x * bs, mby = (uint32_t)r.mb_y * bs;
    const uint32_t ox = (uint32_t)G.off[c][0] + dxx * mbx + dxy * mby + dxx * (uint32_t)L.c;
    const uint32_t oy = (uint32_t)G.off[c][1] + dyx * mbx + dyy * mby + dyx * (uint32_t)L.c;
    const int shift = G.acc + 1, rr = (1 << (2 * G.acc + 1)) - P.no_rnd, ew = P.h_edge >> c, eh = P.v_edge >> c;
    const MpvSrc s = { ref[L.pl], 0, 0, 1, 0, 0, ew, eh };
    const auto t = [&](int x, int y) { return mpv_fetch(P, L.pl, s, x, y); };
    for (int i = 0; i < bs; i++)
        mpv_store(L, i, mpv_gmc_sample(t, ox + dxy * (uint32_t)i, oy + dyy * (uint32_t)i, shift, rr, ew, eh), 0);
}

// ff_mpv_motion for a record of an S-VOP: a 16X16 record with mcsel runs gmc1_motion / gmc_motion (mpegvideo_motion.c:834-843) with put
// for each direction it names, every other record the plain body (IL: that of an interlaced picture, FIELD records included)
template <int IL = 0>
__device__ __forceinline__ void mpv_gmc_lane(const MpvMcPic &P, const MpvGmcParams &G, const FFMpvMCRecord &r, int lane)
{
    if (r.mv_type != MPV_MC_16X16 || !r.mcsel) {
        mpv_mc_lane<1, IL>(P, r, lane);
        return;
    }
    MpvLane L;
    L.pl = lane < 16 ? 0 : 1 + ((lane - 16) >> 3);
    L.c = L.pl ? (lane & 7) : lane;
    const int bs = L.pl ? 8 : 16;
    L.dls = P.ls[L.pl != 0];
    L.dcol = P.dest[L.pl] + (ptrdiff_t)r.mb_y * bs * L.dls + r.mb_x * bs + L.c;
    for (int dir = 0; dir < 2; dir++) {
        if (!((r.mv_dir >> dir) & 1)) continue;
        if (G.pts == 1) mpv_gmc1_motion(P, G, L, r, P.ref[dir]);
        else            mpv_gmc_motion(P, G, L, r, P.ref[dir]);
    }
}

}  // namespace avb
