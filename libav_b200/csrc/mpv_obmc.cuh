// libav_b200/csrc/mpv_obmc.cuh -- H.263 overlapped block motion compensation: apply_obmc (libavcodec/mpegvideo_motion.c:643-728) for one
// macroblock, one lane per destination column like mpv_mc_block.cuh, whose fetch / store / chroma_4mv helpers it reuses.  A separate kernel
// (mpv_obmc_kernel in mpv_mc.cu) runs it, so the plain MC kernel is unchanged.  Lanes never communicate: tests/hostsim/ runs the body.
#pragma once
#include "mpv_mc_block.cuh"

namespace avb {

// put_obmc's weights (mpegvideo_motion.c:407-463; H.263 Annex F): top | left << 2 | right << 4 | bottom << 6 for row y, column x of an
// 8x8 block at index 8 * y + x; the middle weight is 8 minus the others
static const uint8_t mpv_obmc_weights[64] = {
#define W(t, l, r, b) (uint8_t)((t) | (l) << 2 | (r) << 4 | (b) << 6)
    W(2, 2, 0, 0), W(2, 1, 0, 0), W(2, 1, 0, 0), W(2, 1, 0, 0), W(2, 0, 1, 0), W(2, 0, 1, 0), W(2, 0, 1, 0), W(2, 0, 2, 0),
    W(1, 2, 0, 0), W(1, 2, 0, 0), W(2, 1, 0, 0), W(2, 1, 0, 0), W(2, 0, 1, 0), W(2, 0, 1, 0), W(1, 0, 2, 0), W(1, 0, 2, 0),
    W(1, 2, 0, 0), W(1, 2, 0, 0), W(1, 1, 0, 0), W(1, 1, 0, 0), W(1, 0, 1, 0), W(1, 0, 1, 0), W(1, 0, 2, 0), W(1, 0, 2, 0),
    W(1, 2, 0, 0), W(1, 2, 0, 0), W(1, 1, 0, 0), W(1, 1, 0, 0), W(1, 0, 1, 0), W(1, 0, 1, 0), W(1, 0, 2, 0), W(1, 0, 2, 0),
    W(0, 2, 0, 1), W(0, 2, 0, 1), W(0, 1, 0, 1), W(0, 1, 0, 1), W(0, 0, 1, 1), W(0, 0, 1, 1), W(0, 0, 2, 1), W(0, 0, 2, 1),
    W(0, 2, 0, 1), W(0, 2, 0, 1), W(0, 1, 0, 1), W(0, 1, 0, 1), W(0, 0, 1, 1), W(0, 0, 1, 1), W(0, 0, 2, 1), W(0, 0, 2, 1),
    W(0, 2, 0, 1), W(0, 2, 0, 1), W(0, 1, 0, 2), W(0, 1, 0, 2), W(0, 0, 1, 2), W(0, 0, 1, 2), W(0, 0, 2, 1), W(0, 0, 2, 1),
    W(0, 2, 0, 2), W(0, 1, 0, 2), W(0, 1, 0, 2), W(0, 1, 0, 2), W(0, 0, 1, 2), W(0, 0, 1, 2), W(0, 0, 1, 2), W(0, 0, 2, 2),
#undef W
};

// sample (j, i) of hpel_motion's 8x8 prediction (mpegvideo_motion.c:192-224) for vector (mx, my) of the block at (x0, y0): the position
// clipped to [-16, width] x [-16, height] with the half-sample bit dropped at the clip, clamped addressing where the C code emulates
__device__ __forceinline__ int mpv_obmc_sample(const MpvMcPic &P, int x0, int y0, int mx, int my, int j, int i, int no_rnd)
{
    int dxy = 0;
    const int sx = min(max(x0 + (mx >> 1), -16), P.width), sy = min(max(y0 + (my >> 1), -16), P.height);
    if (sx != P.width) dxy |= mx & 1;
    if (sy != P.height) dxy |= (my & 1) << 1;
    const int emu = (unsigned)sx > (unsigned)max(P.h_edge - (mx & 1) - 8, 0) || (unsigned)sy > (unsigned)max(P.v_edge - (my & 1) - 8, 0);
    const MpvSrc s = { P.ref[0][0], sx, sy, 1, 0, emu, P.h_edge, P.v_edge };
    const int a = mpv_fetch(P, 0, s, j, i);
    if (dxy == 0) return a;
    if (dxy == 1) return (a + mpv_fetch(P, 0, s, j + 1, i) + 1 - no_rnd) >> 1;
    if (dxy == 2) return (a + mpv_fetch(P, 0, s, j, i + 1) + 1 - no_rnd) >> 1;
    return (a + mpv_fetch(P, 0, s, j + 1, i) + mpv_fetch(P, 0, s, j, i + 1) + mpv_fetch(P, 0, s, j + 1, i + 1) + 2 - no_rnd) >> 2;
}

// the record the OBMC kernel takes: a plain-MC record it takes, forward only (apply_obmc predicts from last_picture with put)
__device__ __forceinline__ int mpv_obmc_reject(const MpvMcPic &P, const FFMpvMCRecord &r)
{
    return mpv_mc_reject(P, r) ? 1 : (r.mv_dir & 3) != 1 ? 4 : 0;
}

// apply_obmc for the lane's column: mv_cache of :653-700 (neighbours outside the picture or intra replaced by the own vectors, the row
// below always the own lower row), the four luma blocks as put_obmc sums, then chroma_4mv_motion with the sum of the own vectors
__device__ __forceinline__ void mpv_obmc_lane(const MpvMcPic &P, const FFMpvMCRecord &r, const FFMpvOBMCRecord &o, const uint8_t *wt, int lane)
{
    MpvLane L;
    L.pl = lane < 16 ? 0 : 1 + ((lane - 16) >> 3);
    L.c = L.pl ? (lane & 7) : lane;
    const int bs = L.pl ? 8 : 16;
    L.dls = P.ls[L.pl != 0];
    L.dcol = P.dest[L.pl] + (ptrdiff_t)r.mb_y * bs * L.dls + r.mb_x * bs + L.c;
    const int no_rnd = P.no_rnd;
    int16_t c[4][4][2];
    for (int k = 0; k < 2; k++) {
        for (int i = 0; i < 2; i++) c[1][1 + i][k] = o.mv[i][k], c[2][1 + i][k] = o.mv[2 + i][k], c[3][1 + i][k] = o.mv[2 + i][k];
        const bool top = r.mb_y > 0 && !(o.mb_type_top & 7), left = r.mb_x > 0 && !(o.mb_type_left & 7);
        const bool right = r.mb_x + 1 < P.mb_w && !(o.mb_type_right & 7);        // IS_INTRA (mpegutils.h:78)
        for (int i = 0; i < 2; i++) {
            c[0][1 + i][k] = top ? o.top[i][k] : c[1][1 + i][k];
            c[1 + i][0][k] = left ? o.left[i][k] : c[1 + i][1][k];
            c[1 + i][3][k] = right ? o.right[i][k] : c[1 + i][2][k];
        }
    }
    if (L.pl == 0) {
        for (int y = 0; y < 16; y++) {
            const int i = (L.c >> 3) + 2 * (y >> 3), bx = L.c & 7, by = y & 7, cx = (i & 1) + 1, cy = (i >> 1) + 1;
            const int w = wt[8 * by + bx], t = w & 3, l = (w >> 2) & 3, rr = (w >> 4) & 3, b = w >> 6, m = 8 - t - l - rr - b;
            const int x0 = r.mb_x * 16 + (i & 1) * 8, y0 = r.mb_y * 16 + (i >> 1) * 8;
            int sum = m * mpv_obmc_sample(P, x0, y0, c[cy][cx][0], c[cy][cx][1], bx, by, no_rnd);
            if (t) sum += t * mpv_obmc_sample(P, x0, y0, c[cy - 1][cx][0], c[cy - 1][cx][1], bx, by, no_rnd);
            if (b) sum += b * mpv_obmc_sample(P, x0, y0, c[cy + 1][cx][0], c[cy + 1][cx][1], bx, by, no_rnd);
            if (l) sum += l * mpv_obmc_sample(P, x0, y0, c[cy][cx - 1][0], c[cy][cx - 1][1], bx, by, no_rnd);
            if (rr) sum += rr * mpv_obmc_sample(P, x0, y0, c[cy][cx + 1][0], c[cy][cx + 1][1], bx, by, no_rnd);
            mpv_store(L, y, (sum + 4) >> 3, 0);
        }
    } else {
        const int mx = o.mv[0][0] + o.mv[1][0] + o.mv[2][0] + o.mv[3][0], my = o.mv[0][1] + o.mv[1][1] + o.mv[2][1] + o.mv[3][1];
        mpv_chroma_4mv(P, L, r, P.ref[0], no_rnd, 0, mx, my);
    }
}

}  // namespace avb
