// libav_b200/csrc/h263_lf.cuh -- the H.263 deblocking filter (Annex J): H263DSPContext's two edge filters (libavcodec/h263dsp.c:31-115)
// and ff_h263_loop_filter (libavcodec/h263.c:135-220) run for every macroblock of whole pictures.  Device code and the kernels' views
// only, with internal linkage, so any translation unit may include it: the host entry points live in mpv_mc.cu (the picture filter and
// the flush point that ends with it) and h263dsp.cu (the slots).  tests/hostsim/ compiles it as host C++ through mpv_mc.cu.
//
// The picture filter rests on an ordering fact of the serial driver.  A horizontal-edge filter (h263_v_loop_filter, rows 8m-2 .. 8m+1)
// that shares a sample with a vertical-edge filter (h263_h_loop_filter, columns 8m-2 .. 8m+1) always runs before it, and two filters of
// the same direction never share a sample.  So the serial result equals: every horizontal edge, then every vertical edge, each edge's qp
// a function of its two macroblocks alone (DESIGN.md section 5).  One thread owns the 8 x 8 tile centred on the crossing of horizontal
// edge 8j and vertical edge 8k of one plane: every sample of the four lines of both edges' segments in it lies inside it, so it reads the
// tile, filters the horizontal edge, then the vertical one, and writes the tile back.  The tiles partition the plane and no thread reads
// a sample another writes: no halo, no barrier, each byte crossed once each way.
#pragma once
#include "common.cuh"
#include "../../include/avdsp_b200.h"

namespace avb {

enum { H263_MB_TYPE_SKIP = 1 << 11 };     // MB_TYPE_SKIP (mpegutils.h:62)
enum { H263_LF_PICS_PER_LAUNCH = 16 };

// ff_h263_loop_filter_strength (h263dsp.c:26-29)
static const uint8_t h263_lf_strength_tab[32] = {
    0, 1, 1, 2, 2, 3, 3, 4, 4, 4, 5, 5, 6, 6, 7, 7, 7, 8, 8, 8, 9, 9, 9, 10, 10, 10, 11, 11, 11, 12, 12, 12
};

// one line across an edge: p0 p1 | p2 p3 (h263dsp.c:36-71).  `/` truncates towards zero as in C; p1 / p2 are clipped only when bit 8
// is set.
__host__ __device__ __forceinline__ void h263_lf_line(int &p0, int &p1, int &p2, int &p3, int strength)
{
    const int d = (p0 - p3 + 4 * (p2 - p1)) / 8;
    const int d1 = d < -2 * strength ? 0 : d < -strength ? -2 * strength - d : d < strength ? d : d < 2 * strength ? 2 * strength - d : 0;
    int q1 = p1 + d1, q2 = p2 - d1;
    if (q1 & 256) q1 = ~(q1 >> 31);
    if (q2 & 256) q2 = ~(q2 >> 31);
    const int ad1 = (d1 < 0 ? -d1 : d1) >> 1;
    int d2 = (p0 - p3) / 4;
    d2 = d2 < -ad1 ? -ad1 : d2 > ad1 ? ad1 : d2;
    p0 = (uint8_t)(p0 - d2); p1 = (uint8_t)q1; p2 = (uint8_t)q2; p3 = (uint8_t)(p3 + d2);
}

// H263DSPContext slots as a batch of one: thread t filters line t of the 8 (vert 1: h263_h_loop_filter, a vertical edge between columns
// -1 and 0, line = row t; vert 0: h263_v_loop_filter, a horizontal edge between rows -1 and 0, line = column t)
static __global__ void __launch_bounds__(32) h263_lf_slot_kernel(uint8_t *src, int stride, int strength, int vert)
{
    const int t = threadIdx.x;
    if (t >= 8) return;
    uint8_t *o = vert ? src + t * stride : src + t;
    const int s = vert ? 1 : stride;
    int p0 = o[-2 * s], p1 = o[-s], p2 = o[0], p3 = o[s];
    h263_lf_line(p0, p1, p2, p3, strength);
    o[-2 * s] = (uint8_t)p0; o[-s] = (uint8_t)p1; o[0] = (uint8_t)p2; o[s] = (uint8_t)p3;
}

// what the kernel reads of one picture
struct H263LfPic {
    uint8_t *data[3];
    int ls[2];                   // linesize, uvlinesize
    int mb_w, mb_h, mb_stride;
    const uint32_t *mb_type;
    const int8_t *qscale;
    uint8_t strength[2][32];     // [0][qp]: luma strength; [1][qp]: the strength of chroma_qscale_table[qp]
};

struct H263LfLaunch {
    H263LfPic pic[H263_LF_PICS_PER_LAUNCH];
};

// qp_c of macroblock (x, y): 0 for a skipped macroblock (and for a qscale outside 1..31, which the decoder never stores)
__device__ __forceinline__ int h263_lf_qpc(const H263LfPic &P, int x, int y)
{
    const int i = x + y * P.mb_stride;
    const int q = P.qscale[i];
    return (P.mb_type[i] & H263_MB_TYPE_SKIP) || q < 1 || q > 31 ? 0 : q;
}

// qp of the edge in front of 8-sample block a (a >= 1) along one axis, in macroblock o of the other axis.  In luma an odd block starts
// inside its macroblock (qp_c of that macroblock); everywhere else the edge is a macroblock boundary: qp_c of the macroblock after it,
// or, when that is 0, of the one before it.
__device__ __forceinline__ int h263_lf_edge_qp(const H263LfPic &P, int horiz, int luma, int a, int o)
{
    const int m = a >> luma;
    int q = horiz ? h263_lf_qpc(P, o, m) : h263_lf_qpc(P, m, o);
    if (!q && !(luma && (a & 1))) q = horiz ? h263_lf_qpc(P, o, m - 1) : h263_lf_qpc(P, m - 1, o);
    return q;
}

// 4 samples at p (p % 4 == 0 when aligned); bytes little-endian in the word
__device__ __forceinline__ uint32_t h263_lf_ld4(const uint8_t *p, bool aligned)
{
    if (aligned) return *reinterpret_cast<const uint32_t *>(p);
    return (uint32_t)p[0] | (uint32_t)p[1] << 8 | (uint32_t)p[2] << 16 | (uint32_t)p[3] << 24;
}
__device__ __forceinline__ void h263_lf_st4(uint8_t *p, uint32_t v, bool aligned)
{
    if (aligned) { *reinterpret_cast<uint32_t *>(p) = v; return; }
    p[0] = (uint8_t)v; p[1] = (uint8_t)(v >> 8); p[2] = (uint8_t)(v >> 16); p[3] = (uint8_t)(v >> 24);
}

// the 8 x 8 tile rows [8j-4, 8j+4) x columns [8k-4, 8k+4) of plane pl, centred on the crossing of the horizontal edge at row 8j and the
// vertical edge at column 8k: both edges' four lines lie wholly inside it, so the tile is filtered from its own samples alone.  A tile
// half lies wholly inside or wholly outside the plane (its sides are multiples of 8), so only whole halves are masked.
__device__ __forceinline__ void h263_lf_tile(const H263LfPic &P, int pl, int j, int k)
{
    const int luma = pl == 0, nbx = P.mb_w << luma, nby = P.mb_h << luma;       // the plane in 8-sample blocks across / down
    const ptrdiff_t ls = P.ls[!luma];
    const bool aligned = ((((uintptr_t)P.data[pl]) | (uintptr_t)ls) & 3) == 0;
    uint8_t *base = P.data[pl] + (ptrdiff_t)(8 * j - 4) * ls + 8 * k - 4;
    const bool hl = k > 0, hr = k < nbx, ht = j > 0, hb = j < nby;   // the tile's left / right / top / bottom halves exist
    const int r0 = ht ? 0 : 4, r1 = hb ? 8 : 4;
    const uint8_t *str = P.strength[!luma];

    int v[8][8];
#pragma unroll
    for (int r = 0; r < 8; r++) {
        uint32_t a = 0, b = 0;
        if (r >= r0 && r < r1) {
            if (hl) a = h263_lf_ld4(base + r * ls, aligned);
            if (hr) b = h263_lf_ld4(base + r * ls + 4, aligned);
        }
#pragma unroll
        for (int c = 0; c < 4; c++) { v[r][c] = (a >> (8 * c)) & 255; v[r][c + 4] = (b >> (8 * c)) & 255; }
    }
    // the horizontal edge at row 8j (tile rows 2 .. 5), then the vertical edge at column 8k (tile columns 2 .. 5)
    if (ht && hb) {
#pragma unroll
        for (int h = 0; h < 2; h++) {
            if (!(h ? hr : hl)) continue;
            const int q = h263_lf_edge_qp(P, 1, luma, j, (k - 1 + h) >> luma);
            if (!q) continue;
            const int s = str[q];
#pragma unroll
            for (int c = 4 * h; c < 4 * h + 4; c++) h263_lf_line(v[2][c], v[3][c], v[4][c], v[5][c], s);
        }
    }
    if (hl && hr) {
#pragma unroll
        for (int h = 0; h < 2; h++) {
            if (!(h ? hb : ht)) continue;
            const int q = h263_lf_edge_qp(P, 0, luma, k, (j - 1 + h) >> luma);
            if (!q) continue;
            const int s = str[q];
#pragma unroll
            for (int r = 4 * h; r < 4 * h + 4; r++) h263_lf_line(v[r][2], v[r][3], v[r][4], v[r][5], s);
        }
    }
#pragma unroll
    for (int r = 0; r < 8; r++) {
        if (r < r0 || r >= r1) continue;
        uint32_t a = 0, b = 0;
#pragma unroll
        for (int c = 0; c < 4; c++) { a |= (uint32_t)v[r][c] << (8 * c); b |= (uint32_t)v[r][c + 4] << (8 * c); }
        if (hl) h263_lf_st4(base + r * ls, a, aligned);
        if (hr) h263_lf_st4(base + r * ls + 4, b, aligned);
    }
}

// grid: x over the tiles of the largest plane, y = 3 * picture + plane
static __global__ void __launch_bounds__(128) h263_lf_kernel(const __grid_constant__ H263LfLaunch L)
{
    const int pi = blockIdx.y / 3, pl = blockIdx.y % 3;
    const H263LfPic &P = L.pic[pi];
    const int luma = pl == 0, nw = (P.mb_w << luma) + 1, nh = (P.mb_h << luma) + 1;
    const unsigned i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= (unsigned)(nw * nh)) return;
    h263_lf_tile(P, pl, (int)(i / nw), (int)(i % nw));
}

}  // namespace avb
