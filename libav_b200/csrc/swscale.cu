// libav_b200/csrc/swscale.cu -- libswscale's scaler for yuv420p sources on sm_90a.
//
// Replaces, bit-exactly (SWS_ACCURATE_RND | SWS_BITEXACT semantics), the C slots that swscale() drives
// (libswscale/swscale.c:343-721):
//   hyScale / hcScale = hScale8To15_c                       libswscale/swscale.c:133-147
//   yuv2packedX/2/1   = yuv2rgb24_{X,2,1}_c                 libswscale/output.c:936-1110 (+ write :853-866)
//   yuv2planeX / yuv2plane1 (8 bit)                         libswscale/output.c:242-265
//   line scheduling + vertical edge replication             libswscale/swscale.c:450-616
// The yuv->rgb look-up tables (libswscale/yuv2rgb.c:633-658, :850-863) are never materialised: the table
// entry ytab[Y + off(U,V)] == clip_u8((cy * (Y + off) + k1) >> 16) is evaluated arithmetically, which is
// exact for every in-range index and removes 5 scattered byte/word gathers per pixel.
//
// Two execution shapes:
//   FUSED (the 4K benchmark geometry: same-size yuv420p -> rgb24/bgr24, bicubic): the horizontal filters are
//     the identity and vLum is {4096}, so one kernel reads Y,U,V bytes and writes RGB: 1.5 B in + 3 B out per
//     pixel, nothing else touches HBM.  A thread owns 8 pixels x 2 rows (one chroma window, two phases).
//   GENERAL (any other geometry): hscale pass into 15-bit int16 planes, then a vertical+output pass that
//     follows the reference's X / 2 / 1 function selection (swscale.c:659-682) line for line.
#include "common.cuh"
#include "scratch.h"
#include "sws_filter.h"
#include "../../include/avdsp_b200.h"
#include <new>
#include <vector>
#include "sws_dev.cuh"
#include "sws_fused.h"
#include <algorithm>
#include <limits.h>
#include <string.h>

namespace avb {

struct SwsDev {                       // kernel-side view of a context (passed by value)
    int srcW, srcH, dstW, dstH, chrSrcW, chrSrcH, chrDstW, chrDstH;
    int hLumSize, hChrSize, vLumSize, vChrSize;
    const int16_t *hLumF, *hChrF, *vLumF, *vChrF;
    const int32_t *hLumP, *hChrP, *vLumP, *vChrP;
    RgbConstants k;
    int bgr;
    int full;                         // SWS_FULL_CHR_H_INT: one chroma sample per output pixel, yuv2rgb24_full_X_c
    int dstBits;                      // planar destinations: 8, 9 / 10 (16-bit samples, yuv2planeX_10_c) or 16 (yuv2planeX_16_c)
    int pk422;                        // packed 4:2:2 destination: 1 yuyv422, 2 uyvy422 (yuv2422_X / _2 / _1, output.c:448-576)
    int rgb16;                        // 15 / 16 / 12-bpp destination: 1 rgb565 2 bgr565 3 rgb555 4 bgr555 5 rgb444 6 bgr444, + 8 big-endian (yuv2rgb_write, output.c:869-902)
    int srcGray;                      // gray8 source: chroma lines are the constant the reference's line buffers hold (bytes of 64)
    int rgb48;                        // 48-bit destination: 1 rgb48 2 bgr48, + 8 big-endian (yuv2rgb48_X / _2 / _1_c_template, output.c:584-760; yuv2rgb_c_48, yuv2rgb.c:106-236)
    int chrStep;                      // 2 for an nv12 / nv21 destination: the chroma planes interleave in one plane (yuv2nv12cX_c, output.c:267-303)
    int dstBE;                        // 16-bit samples are stored big-endian (AV_WB16 in output_pixel, output.c:124-133,176-181)
    int srcBits, srcBE;               // 9 / 10 / 16-bit planar sources: 16-bit words (byte-swapped when big-endian), hScale16To15_c; else 8
    int dither;                       // those sources dither their 8-bit planar outputs (should_dither, swscale.c:389-390,553-556)
};

// ---------------------------------------------------------------------------------------------------
// FUSED kernel: horizontal identity, vLum identity, 4-tap vertical chroma.
// ---------------------------------------------------------------------------------------------------
// (FusedArgs: sws_fused.h)

// one output row of 8 pixels from 8 luma bytes and 4 already filtered (U,V) pairs -> 6 packed words
__device__ __forceinline__ void rgb_row8(uint2 yy, const int (&U)[4], const int (&V)[4], const RgbConstants &k, int bgr,
                                         uint32_t (&out)[6])
{
    int r[8], g[8], b[8];
#pragma unroll
    for (int c = 0; c < 4; c++) {
        int u = U[c], v = V[c];
        if ((u | v) & 0x100) { u = clip_u8(u); v = clip_u8(v); }     // luma is a byte: only chroma can flag
        ChromaTerms t = chroma_terms(u, v, k);
        int tr = bgr ? t.tb : t.tr, tb = bgr ? t.tr : t.tb;
#pragma unroll
        for (int s = 0; s < 2; s++) {
            int p = 2 * c + s;
            int Y = byte_of(p < 4 ? yy.x : yy.y, p & 3);
            r[p] = (k.cy * Y + tr) >> 16;
            g[p] = (k.cy * Y + t.tg) >> 16;
            b[p] = (k.cy * Y + tb) >> 16;
        }
    }
#pragma unroll
    for (int h = 0; h < 2; h++) {
        int o = 4 * h;
        out[3 * h + 0] = pack4_sat_u8(r[o], g[o], b[o], r[o + 1]);
        out[3 * h + 1] = pack4_sat_u8(g[o + 1], b[o + 1], r[o + 2], g[o + 2]);
        out[3 * h + 2] = pack4_sat_u8(b[o + 2], r[o + 3], g[o + 3], b[o + 3]);
    }
}

__device__ __forceinline__ int clampi(int v, int lo, int hi) { return min(max(v, lo), hi); }

template <bool ALIGNED>
__global__ void __launch_bounds__(256)
sws_fused_rgb24_kernel(SwsDev p, FusedArgs a)
{
    const int gx = blockIdx.x * 32 + threadIdx.x;            // group of 8 pixels
    const int rp = blockIdx.y * 8 + threadIdx.y;             // row pair
    const int x0 = gx * 8, y0 = rp * 2;
    if (x0 >= p.dstW || y0 >= p.dstH) return;
    const size_t f = blockIdx.z;
    const uint8_t *Y = a.y + f * a.yFrame, *Uc = a.u + f * a.uFrame, *Vc = a.v + f * a.vFrame;
    uint8_t *D = a.dst + f * a.dstFrame;
    const bool full = ALIGNED && x0 + 8 <= p.dstW;     // vector path; otherwise byte accesses (tails, odd pitches)
    // whole pixel pairs are written like the reference (one pixel past an odd dstW, output.c:947) only when the
    // row pitch has room for it -- rows are concurrent here, the spill must never land in the next row
    const int writeW = ((p.dstW & 1) && a.dstStride >= 3 * (p.dstW + 1)) ? p.dstW + 1 : p.dstW;

    uint32_t uw[4], vw[4];
    int loaded_first = INT_MIN;
#pragma unroll
    for (int ry = 0; ry < 2; ry++) {
        const int y = y0 + ry;
        if (y >= p.dstH) break;
        const int first = max(1 - 4, p.vChrP[y]);            // swscale.c:463
        if (first != loaded_first) {                         // both rows of a pair normally share the window
#pragma unroll
            for (int j = 0; j < 4; j++) {
                int row = clampi(first + j, 0, p.chrSrcH - 1);   // vertical edge replication, swscale.c:592-616
                if (full) {
                    uw[j] = *reinterpret_cast<const uint32_t *>(Uc + (size_t)row * a.uStride + x0 / 2);
                    vw[j] = *reinterpret_cast<const uint32_t *>(Vc + (size_t)row * a.vStride + x0 / 2);
                } else {
                    uint32_t uu = 0, vv = 0;
                    for (int c = 0; c < 4; c++) {
                        int cx = min(x0 / 2 + c, p.chrSrcW - 1);
                        uu |= (uint32_t)Uc[(size_t)row * a.uStride + cx] << (8 * c);
                        vv |= (uint32_t)Vc[(size_t)row * a.vStride + cx] << (8 * c);
                    }
                    uw[j] = uu; vw[j] = vv;
                }
            }
            loaded_first = first;
        }
        const int16_t *cf = p.vChrF + (size_t)y * 4;
        const int c0 = cf[0], c1 = cf[1], c2 = cf[2], c3 = cf[3];
        int U[4], V[4];
#pragma unroll
        for (int c = 0; c < 4; c++) {
            // (2^18 + sum (u << 7) * coef) >> 19  ==  (2^11 + sum u * coef) >> 12
            U[c] = (2048 + byte_of(uw[0], c) * c0 + byte_of(uw[1], c) * c1 + byte_of(uw[2], c) * c2 + byte_of(uw[3], c) * c3) >> 12;
            V[c] = (2048 + byte_of(vw[0], c) * c0 + byte_of(vw[1], c) * c1 + byte_of(vw[2], c) * c2 + byte_of(vw[3], c) * c3) >> 12;
        }
        uint2 yy;
        const uint8_t *yrow = Y + (size_t)y * a.yStride + x0;
        if (full) yy = *reinterpret_cast<const uint2 *>(yrow);
        else {
            yy = make_uint2(0, 0);               // pixels beyond dstW read as 0, like the zeroed line buffer
            for (int c = 0; c < 8 && x0 + c < p.dstW; c++) {
                if (c < 4) yy.x |= (uint32_t)yrow[c] << (8 * c); else yy.y |= (uint32_t)yrow[c] << (8 * (c - 4));
            }
        }
        uint32_t o[6];
        rgb_row8(yy, U, V, p.k, p.bgr, o);
        uint8_t *drow = D + (size_t)y * a.dstStride + (size_t)x0 * 3;
        if (full) {
            uint2 *d2 = reinterpret_cast<uint2 *>(drow);
            d2[0] = make_uint2(o[0], o[1]); d2[1] = make_uint2(o[2], o[3]); d2[2] = make_uint2(o[4], o[5]);
        } else {
            int npx = min(8, writeW - x0);
            for (int c = 0; c < npx * 3; c++) drow[c] = (uint8_t)(o[c >> 2] >> (8 * (c & 3)));
        }
    }
}

// ---------------------------------------------------------------------------------------------------
// FUSED kernel, interior fast path (LDG variant; the TMA-staged kernel of sws_fused_tma.cu runs instead whenever tensor maps can
// describe the planes).  A thread owns 16 pixels x 2 rows (one LDG.128 of luma per row, one LDG.64 per chroma line).
// Preconditions checked on the host (else the kernel above runs): 16-byte aligned planes / pitches, dstW % 16 == 0, dstH even, the
// chroma windows of the two rows of every pair start at most one line apart, and the filter bank cannot push U,V outside (-256, 512)
// -- then clipping each value on its own is identical to the reference's "clip all four if any has bit 8 set" (output.c:966-971)
// because an in-range value is unchanged by av_clip_uint8.
// The 4 chroma lines of a column are byte-transposed into one word
// (2 PRMT per column instead of 4-5 byte extracts -- the 16-lane ALU pipe is the limiter of these kernels) and the 4-tap
// FIR becomes two IDP4A (coefficient = 256 * hi + lo, lo unsigned byte, hi signed byte) plus one IMAD.  Per row pair the
// packed taps, the fifth tap and the first chroma line come from a host-built table (SwsPairTaps).
struct SwsPairTaps { uint32_t lo0, hi0, lo1, hi1; int tap4; int first; int pad0, pad1; };   // 32 bytes per row pair

#ifdef AVB_HOSTSIM      // tests/hostsim/: the two dot-product instructions spelled out
inline int dp4a_uu(uint32_t a, uint32_t b, int c) { for (int k = 0; k < 4; k++) c += (int)((a >> (8 * k)) & 255) * (int)((b >> (8 * k)) & 255); return c; }
inline int dp4a_us(uint32_t a, uint32_t b, int c) { for (int k = 0; k < 4; k++) c += (int)((a >> (8 * k)) & 255) * (int)(int8_t)((b >> (8 * k)) & 255); return c; }
#else
__device__ __forceinline__ int dp4a_uu(uint32_t a, uint32_t b, int c)
{ int d; asm("dp4a.u32.u32 %0, %1, %2, %3;" : "=r"(d) : "r"(a), "r"(b), "r"(c)); return d; }
__device__ __forceinline__ int dp4a_us(uint32_t a, uint32_t b, int c)
{ int d; asm("dp4a.u32.s32 %0, %1, %2, %3;" : "=r"(d) : "r"(a), "r"(b), "r"(c)); return d; }
#endif

template <bool BGR>
__global__ void __launch_bounds__(128)
sws_fused_rgb24_v3_kernel(SwsDev p, FusedArgs a, const SwsPairTaps *__restrict__ taps)
{
    const int gx = blockIdx.x * 32 + threadIdx.x;            // group of 16 pixels
    const int rp = a.rp0 + blockIdx.y * 4 + threadIdx.y;     // row pair
    if (gx * 16 >= p.dstW || rp >= a.rp1) return;
    const size_t f = blockIdx.z;
    const int y0 = rp * 2;
    const uint8_t *Yp = a.y + f * a.yFrame + (size_t)y0 * a.yStride + gx * 16;
    const uint8_t *Up = a.u + f * a.uFrame + gx * 8, *Vp = a.v + f * a.vFrame + gx * 8;
    uint8_t *D = a.dst + f * a.dstFrame + (size_t)y0 * a.dstStride + gx * 48;

    const uint4 tq = __ldg(reinterpret_cast<const uint4 *>(taps + rp));
    const int2 tz = __ldg(reinterpret_cast<const int2 *>(taps + rp) + 2);
    const int first = tz.y, tap4 = tz.x;
    uint2 u[5], v[5];
#pragma unroll
    for (int j = 0; j < 5; j++) {
        const int row = min(max(first + j, 0), p.chrSrcH - 1);
        u[j] = __ldg(reinterpret_cast<const uint2 *>(Up + (size_t)row * a.uStride));
        v[j] = __ldg(reinterpret_cast<const uint2 *>(Vp + (size_t)row * a.vStride));
    }
    const uint4 yy0 = ldg_stream(Yp), yy1 = ldg_stream(Yp + a.yStride);
    const int cy = p.k.cy, crv = p.k.crv, cgu = p.k.cgu, cgv = p.k.cgv, cbu = p.k.cbu, kr = p.k.kr, kg = p.k.kg, kb = p.k.kb;

    uint32_t o0[12], o1[12];
#pragma unroll
    for (int hq = 0; hq < 2; hq++) {                         // half of the group: 4 chroma columns = 8 pixels
        // 4x4 byte transposes: TU[c] = (line0, line1, line2, line3) of chroma column c
        uint32_t TU[4], TV[4];
        {
            const uint32_t r0 = hq ? u[0].y : u[0].x, r1 = hq ? u[1].y : u[1].x, r2 = hq ? u[2].y : u[2].x, r3 = hq ? u[3].y : u[3].x;
            const uint32_t t0 = __byte_perm(r0, r1, 0x5140), t1 = __byte_perm(r2, r3, 0x5140), t2 = __byte_perm(r0, r1, 0x7362), t3 = __byte_perm(r2, r3, 0x7362);
            TU[0] = __byte_perm(t0, t1, 0x5410); TU[1] = __byte_perm(t0, t1, 0x7632); TU[2] = __byte_perm(t2, t3, 0x5410); TU[3] = __byte_perm(t2, t3, 0x7632);
        }
        {
            const uint32_t r0 = hq ? v[0].y : v[0].x, r1 = hq ? v[1].y : v[1].x, r2 = hq ? v[2].y : v[2].x, r3 = hq ? v[3].y : v[3].x;
            const uint32_t t0 = __byte_perm(r0, r1, 0x5140), t1 = __byte_perm(r2, r3, 0x5140), t2 = __byte_perm(r0, r1, 0x7362), t3 = __byte_perm(r2, r3, 0x7362);
            TV[0] = __byte_perm(t0, t1, 0x5410); TV[1] = __byte_perm(t0, t1, 0x7632); TV[2] = __byte_perm(t2, t3, 0x5410); TV[3] = __byte_perm(t2, t3, 0x7632);
        }
        const uint32_t u4w = hq ? u[4].y : u[4].x, v4w = hq ? v[4].y : v[4].x;
#pragma unroll
        for (int q2 = 0; q2 < 2; q2++) {                     // 4 pixels = 2 chroma columns per step
            const int q = 2 * hq + q2;
            int r0[4], g0[4], b0[4], r1[4], g1[4], b1[4];
#pragma unroll
            for (int e = 0; e < 2; e++) {
                const int c = 2 * q2 + e;                    // chroma column inside this half
                const int u4 = byte_of(u4w, c), v4 = byte_of(v4w, c);
#pragma unroll
                for (int ry = 0; ry < 2; ry++) {
                    const uint32_t lo = ry ? tq.z : tq.x, hi = ry ? tq.w : tq.y;
                    int su = dp4a_us(TU[c], hi, 0) * 256 + dp4a_uu(TU[c], lo, 2048);
                    int sv = dp4a_us(TV[c], hi, 0) * 256 + dp4a_uu(TV[c], lo, 2048);
                    if (ry) { su += u4 * tap4; sv += v4 * tap4; }
                    const int U = sat255(su >> 12), V = sat255(sv >> 12);
                    const int tr = cy * ((V * crv) >> 16) + kr;
                    const int tg = cy * (((U * cgu) >> 16) + ((V * cgv) >> 16)) + kg;
                    const int tb = cy * ((U * cbu) >> 16) + kb;
                    const uint4 yy = ry ? yy1 : yy0;
                    const uint32_t yw = q == 0 ? yy.x : q == 1 ? yy.y : q == 2 ? yy.z : yy.w;
                    const int Ya = cy * byte_of(yw, 2 * e), Yb = cy * byte_of(yw, 2 * e + 1);
                    // keep the 32-bit sums; the >> 16, the clip and the packing happen four values at a time below
                    int *r = ry ? r1 : r0, *g = ry ? g1 : g0, *b = ry ? b1 : b0;
                    r[2 * e] = Ya + (BGR ? tb : tr); g[2 * e] = Ya + tg; b[2 * e] = Ya + (BGR ? tr : tb);
                    r[2 * e + 1] = Yb + (BGR ? tb : tr); g[2 * e + 1] = Yb + tg; b[2 * e + 1] = Yb + (BGR ? tr : tb);
                }
            }
            o0[3 * q + 0] = pack4_hi16_sat(r0[0], g0[0], b0[0], r0[1]);
            o0[3 * q + 1] = pack4_hi16_sat(g0[1], b0[1], r0[2], g0[2]);
            o0[3 * q + 2] = pack4_hi16_sat(b0[2], r0[3], g0[3], b0[3]);
            o1[3 * q + 0] = pack4_hi16_sat(r1[0], g1[0], b1[0], r1[1]);
            o1[3 * q + 1] = pack4_hi16_sat(g1[1], b1[1], r1[2], g1[2]);
            o1[3 * q + 2] = pack4_hi16_sat(b1[2], r1[3], g1[3], b1[3]);
        }
    }
#pragma unroll
    for (int k = 0; k < 3; k++) {
        stg_stream(D + 16 * k, make_uint4(o0[4 * k], o0[4 * k + 1], o0[4 * k + 2], o0[4 * k + 3]));
        stg_stream(D + a.dstStride + 16 * k, make_uint4(o1[4 * k], o1[4 * k + 1], o1[4 * k + 2], o1[4 * k + 3]));
    }
}

// ---------------------------------------------------------------------------------------------------
// Unscaled table converter: the SwsFunc the reference installs for same-size yuv420p -> rgb24/bgr24 when SWS_ACCURATE_RND
// is NOT set and dstH is even (swscale_unscaled.c:1051-1055 -> yuv2rgb_c_24_rgb / _bgr, yuv2rgb.c:126-175, :335-372):
// chroma is taken from the nearest sample in both directions (no vertical interpolation), then the same tables.
// It converts dstW & ~1 pixels per row (groups of 8, then 4, then 2: an odd last column is left untouched).
// thread = one chroma sample = 2x2 pixels.
__global__ void __launch_bounds__(256)
sws_unscaled_yuv2rgb24_kernel(SwsDev p, FusedArgs a)
{
    const int cx = blockIdx.x * blockDim.x + threadIdx.x, cyy = blockIdx.y;
    if (cx >= (p.dstW >> 1) || cyy >= (p.dstH >> 1)) return;
    const size_t f = blockIdx.z;
    const int U = a.u[f * a.uFrame + (size_t)cyy * a.uStride + cx], V = a.v[f * a.vFrame + (size_t)cyy * a.vStride + cx];
    const ChromaTerms t = chroma_terms(U, V, p.k);
    const int tr = p.bgr ? t.tb : t.tr, tb = p.bgr ? t.tr : t.tb;
#pragma unroll
    for (int ry = 0; ry < 2; ry++) {
        const uint8_t *yp = a.y + f * a.yFrame + (size_t)(2 * cyy + ry) * a.yStride + 2 * cx;
        uint8_t *d = a.dst + f * a.dstFrame + (size_t)(2 * cyy + ry) * a.dstStride + (p.rgb48 ? 12 : 6) * cx;
#pragma unroll
        for (int e = 0; e < 2; e++) {
            const int Y = yp[e];
            const uint8_t c0 = (uint8_t)clip_u8((p.k.cy * Y + tr) >> 16), c1 = (uint8_t)clip_u8((p.k.cy * Y + t.tg) >> 16), c2 = (uint8_t)clip_u8((p.k.cy * Y + tb) >> 16);
            if (p.rgb48) {              // yuv2rgb_c_48 / _bgr48 (yuv2rgb.c:106-124): the 8-bit table value in both bytes of a component, whatever the endianness
                d[6 * e + 0] = d[6 * e + 1] = c0; d[6 * e + 2] = d[6 * e + 3] = c1; d[6 * e + 4] = d[6 * e + 5] = c2;
            } else { d[3 * e + 0] = c0; d[3 * e + 1] = c1; d[3 * e + 2] = c2; }
        }
    }
}

// ---------------------------------------------------------------------------------------------------
// 48-bit rgb destinations behind swscale() (dstBpc 16): the lines are hScale8To19_c's (swscale.c:62-80,728-741 -- no fast-bilinear line
// functions at that depth) and the output stage is yuv2rgb48_X / _2 / _1_c_template (output.c:593-760) under swscale()'s X / 2 / 1 selection
// (swscale.c:658-683).  One thread = one pixel pair of one output row; it recomputes the horizontal filter for every vertical tap straight
// from the source planes (no line planes: 19-bit lines would be 4 B per sample), all in the wrapping int arithmetic of the C code.
// ---------------------------------------------------------------------------------------------------
__device__ __forceinline__ int h19(const uint8_t *__restrict__ row, const int16_t *__restrict__ f, int pos, int fs)
{
    int v = 0;
    for (int k = 0; k < fs; k++) v += row[pos + k] * f[k];
    return min(v >> 3, (1 << 19) - 1);
}
__device__ __forceinline__ uint32_t clip30(uint32_t a) { return (a & 0xC0000000u) ? ((a >> 31) ? 0u : 0x3FFFFFFFu) : a; }      // av_clip_uintp2(a, 30)
__device__ __forceinline__ void put48(uint8_t *d, int k, uint32_t v30, int be)
{
    const unsigned v = clip30(v30) >> 14;
    d[2 * k + (be ? 1 : 0)] = (uint8_t)v; d[2 * k + (be ? 0 : 1)] = (uint8_t)(v >> 8);
}

__global__ void __launch_bounds__(128)
sws_rgb48_kernel(SwsDev p, FusedArgs a)
{
    const int i = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y;
    if (i >= ((p.dstW + 1) >> 1) || y >= p.dstH) return;
    const size_t f = blockIdx.z;
    const uint8_t *Yp = a.y + f * a.yFrame, *Up = a.u + f * a.uFrame, *Vp = a.v + f * a.vFrame;
    const int fl = p.vLumSize, fc = p.vChrSize;
    const int firstL = max(1 - fl, p.vLumP[y]), firstC = max(1 - fc, p.vChrP[y]);
    const int x0 = 2 * i, x1 = 2 * i + 1;
    const bool has2 = x1 < p.dstW;            // odd width: the pair's second pixel reads the zeroed tail of the line
    const int16_t *hf0 = p.hLumF + (size_t)x0 * p.hLumSize, *hf1 = p.hLumF + (size_t)(has2 ? x1 : x0) * p.hLumSize, *hfc = p.hChrF + (size_t)i * p.hChrSize;
    const int p0 = p.hLumP[x0], p1 = p.hLumP[has2 ? x1 : x0], pc = p.hChrP[i];
    auto L0 = [&](int j) -> uint32_t { return (uint32_t)h19(Yp + (size_t)clampi(firstL + j, 0, p.srcH - 1) * a.yStride, hf0, p0, p.hLumSize); };
    auto L1 = [&](int j) -> uint32_t { return has2 ? (uint32_t)h19(Yp + (size_t)clampi(firstL + j, 0, p.srcH - 1) * a.yStride, hf1, p1, p.hLumSize) : 0u; };
    // (a gray8 source has no chroma lines: the vertical stage reads the bytes of 64 the reference's line buffers were initialised with, 0x40404040 per 19-bit sample)
    auto CU = [&](int j) -> uint32_t { return p.srcGray ? 0x40404040u : (uint32_t)h19(Up + (size_t)clampi(firstC + j, 0, p.chrSrcH - 1) * a.uStride, hfc, pc, p.hChrSize); };
    auto CV = [&](int j) -> uint32_t { return p.srcGray ? 0x40404040u : (uint32_t)h19(Vp + (size_t)clampi(firstC + j, 0, p.chrSrcH - 1) * a.vStride, hfc, pc, p.hChrSize); };
    int Y1, Y2, U, V;
    if (fl == 1 && fc <= 2) {                                  // yuv2rgb48_1_c_template, output.c:694-760
        const int uvalpha = fc == 1 ? 0 : p.vChrF[2 * y + 1];
        Y1 = (int)L0(0) >> 2; Y2 = (int)L1(0) >> 2;
        if (uvalpha < 2048) { U = ((int)CU(0) - (128 << 11)) >> 2; V = ((int)CV(0) - (128 << 11)) >> 2; }
        else                { U = ((int)(CU(0) + CU(1)) - (128 << 12)) >> 3; V = ((int)(CV(0) + CV(1)) - (128 << 12)) >> 3; }
    } else if (fl == 2 && fc == 2) {                           // yuv2rgb48_2_c_template, output.c:652-692
        const uint32_t ya = (uint32_t)(int)p.vLumF[2 * y + 1], ua = (uint32_t)(int)p.vChrF[2 * y + 1], ya1 = 4096u - ya, ua1 = 4096u - ua, bias = (uint32_t)(-128 * (1 << 23));
        Y1 = (int)(L0(0) * ya1 + L0(1) * ya) >> 14;
        Y2 = (int)(L1(0) * ya1 + L1(1) * ya) >> 14;
        U = (int)(CU(0) * ua1 + CU(1) * ua + bias) >> 14;
        V = (int)(CV(0) * ua1 + CV(1) * ua + bias) >> 14;
    } else {                                                   // yuv2rgb48_X_c_template, output.c:593-650
        const int16_t *lf = p.vLumF + (size_t)y * fl, *cf = p.vChrF + (size_t)y * fc;
        uint32_t a1 = (uint32_t)-0x40000000, a2 = a1, au = (uint32_t)(-128 * (1 << 23)), av = au;
        for (int j = 0; j < fl; j++) { a1 += L0(j) * (uint32_t)(int)lf[j]; a2 += L1(j) * (uint32_t)(int)lf[j]; }
        for (int j = 0; j < fc; j++) { au += CU(j) * (uint32_t)(int)cf[j]; av += CV(j) * (uint32_t)(int)cf[j]; }
        Y1 = ((int)a1 >> 14) + 0x10000; Y2 = ((int)a2 >> 14) + 0x10000; U = (int)au >> 14; V = (int)av >> 14;
    }
    const RgbConstants &k = p.k;
    const uint32_t y1 = (uint32_t)(Y1 - k.fy_offset) * (uint32_t)k.fy_coeff + (1u << 13), y2 = (uint32_t)(Y2 - k.fy_offset) * (uint32_t)k.fy_coeff + (1u << 13);
    const uint32_t R = (uint32_t)V * (uint32_t)k.fv2r, G = (uint32_t)V * (uint32_t)k.fv2g + (uint32_t)U * (uint32_t)k.fu2g, B = (uint32_t)U * (uint32_t)k.fu2b;
    const int bgr = (p.rgb48 & 7) == 2, be = p.rgb48 & 8;
    uint8_t *d = a.dst + f * a.dstFrame + (size_t)y * a.dstStride + (size_t)i * 12;
    put48(d, 0, (bgr ? B : R) + y1, be); put48(d, 1, G + y1, be); put48(d, 2, (bgr ? R : B) + y1, be);
    if (has2 || a.dstStride >= 6 * (p.dstW + 1)) { put48(d, 3, (bgr ? B : R) + y2, be); put48(d, 4, G + y2, be); put48(d, 5, (bgr ? R : B) + y2, be); }
}

// ---------------------------------------------------------------------------------------------------
// GENERAL path, pass 1: hScale8To15 (swscale.c:133-147) for one plane; thread = (column, row)
// ---------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256)
sws_hscale8to15_kernel(const uint8_t *__restrict__ src, int srcStride, int16_t *__restrict__ dst, int dstStridePx,
                       const int16_t *__restrict__ filter, const int32_t *__restrict__ pos, int fs, int dstW, int rows)
{
    int i = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y;
    if (i >= dstW || y >= rows) return;
    const uint8_t *s = src + (size_t)y * srcStride + pos[i];
    const int16_t *f = filter + (size_t)i * fs;
    int val = 0;
    for (int j = 0; j < fs; j++) val += (int)s[j] * f[j];
    dst[(size_t)y * dstStridePx + i] = (int16_t)min(val >> 7, (1 << 15) - 1);
}

// hyscale_fast_c / hcscale_fast_c (swscale.c:238-250, :286-299), selected by SWS_FAST_BILINEAR instead of the filter
// bank.  The reference reads src[xx + 1] one byte past the last source pixel; that byte is defined here as a copy
// of the last pixel (documented deviation: the reference's value is whatever follows the row in memory).
__global__ void __launch_bounds__(256)
sws_hscale_fast_kernel(const uint8_t *__restrict__ src, int srcStride, int16_t *__restrict__ dst, int dstStridePx,
                       int srcW, int dstW, int rows, unsigned xInc, int chroma)
{
    int i = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y;
    if (i >= dstW || y >= rows) return;
    unsigned xpos = (unsigned)i * xInc, xx = xpos >> 16, xa = (xpos & 0xFFFF) >> 9;
    const uint8_t *s = src + (size_t)y * srcStride;
    int a = s[xx], b = s[min(xx + 1, (unsigned)srcW - 1)];
    dst[(size_t)y * dstStridePx + i] = (int16_t)(chroma ? a * (int)(xa ^ 127) + b * (int)xa : (a << 7) + (b - a) * (int)xa);
}

__device__ __forceinline__ int line_index(int first, int j, int srcH) { return clampi(first + j, 0, srcH - 1); }

// pass 2 for packed RGB: thread = (pixel pair, output row); X / 2 / 1 selection as swscale.c:659-682
__global__ void __launch_bounds__(256)
sws_vscale_rgb24_kernel(SwsDev p, const int16_t *__restrict__ lum, const int16_t *__restrict__ chrU,
                        const int16_t *__restrict__ chrV, int lumStride, int chrStride, uint8_t *__restrict__ dst,
                        int dstStride)
{
    const int i = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y;
    if (i >= ((p.dstW + 1) >> 1) || y >= p.dstH) return;
    const int fl = p.vLumSize, fc = p.vChrSize;
    const int firstL = max(1 - fl, p.vLumP[y]), firstC = max(1 - fc, p.vChrP[y]);
    const bool has2 = 2 * i + 1 < p.dstW;     // odd width: the second pixel of the last pair reads the zeroed tail
    int Y1, Y2, U, V;
    auto L = [&](int j, int x) -> int { return x < p.dstW ? lum[(size_t)line_index(firstL, j, p.srcH) * lumStride + x] : 0; };
    auto CU = [&](int j) -> int { return chrU[(size_t)line_index(firstC, j, p.chrSrcH) * chrStride + i]; };
    auto CV = [&](int j) -> int { return chrV[(size_t)line_index(firstC, j, p.chrSrcH) * chrStride + i]; };
    if (fl == 1 && fc <= 2) {                                  // yuv2rgb24_1_c, output.c:1042-1110
        int uvalpha = fc == 1 ? 0 : p.vChrF[2 * y + 1];
        Y1 = L(0, 2 * i) >> 7; Y2 = L(0, 2 * i + 1) >> 7;
        if (uvalpha < 2048) { U = CU(0) >> 7; V = CV(0) >> 7; }
        else                { U = (CU(0) + CU(1)) >> 8; V = (CV(0) + CV(1)) >> 8; }
        Y1 = clip_u8(Y1); Y2 = clip_u8(Y2); U = clip_u8(U); V = clip_u8(V);
    } else if (fl == 2 && fc == 2) {                           // yuv2rgb24_2_c, output.c:997-1040
        int ya = p.vLumF[2 * y + 1], ua = p.vChrF[2 * y + 1], ya1 = 4096 - ya, ua1 = 4096 - ua;
        Y1 = (L(0, 2 * i) * ya1 + L(1, 2 * i) * ya) >> 19;
        Y2 = (L(0, 2 * i + 1) * ya1 + L(1, 2 * i + 1) * ya) >> 19;
        U = (CU(0) * ua1 + CU(1) * ua) >> 19;
        V = (CV(0) * ua1 + CV(1) * ua) >> 19;
        Y1 = clip_u8(Y1); Y2 = clip_u8(Y2); U = clip_u8(U); V = clip_u8(V);
    } else {                                                   // yuv2rgb24_X_c, output.c:936-995
        const int16_t *lf = p.vLumF + (size_t)y * fl, *cf = p.vChrF + (size_t)y * fc;
        Y1 = Y2 = U = V = 1 << 18;
        for (int j = 0; j < fl; j++) { Y1 += L(j, 2 * i) * lf[j]; Y2 += L(j, 2 * i + 1) * lf[j]; }
        for (int j = 0; j < fc; j++) { U += CU(j) * cf[j]; V += CV(j) * cf[j]; }
        Y1 >>= 19; Y2 >>= 19; U >>= 19; V >>= 19;
        clip_if_flagged(Y1, Y2, U, V);
    }
    if (p.pk422) {             // the same four values, stored instead of converted (output_pixels, output.c:448-467)
        uint8_t *d = dst + (size_t)y * dstStride + (size_t)i * 4;
        const bool room = has2 || dstStride >= 2 * (p.dstW + 1);      // odd width: the pair's second half needs room in the row
        if (p.pk422 == 1) { d[0] = (uint8_t)Y1; d[1] = (uint8_t)U; if (room) { d[2] = (uint8_t)Y2; d[3] = (uint8_t)V; } }
        else              { d[0] = (uint8_t)U; d[1] = (uint8_t)Y1; if (room) { d[2] = (uint8_t)V; d[3] = (uint8_t)Y2; } }
        return;
    }
    ChromaTerms t = chroma_terms(U, V, p.k);
    if (p.rgb16) {
        // yuv2rgb_write for 565 / 555 / 444 (output.c:869-902): r[Y + dr] + g[Y + dg] + b[Y + db] with the 2 x 2 (4 x 4 for 444) ordered
        // dither added to the table INDEX; the tables hold the 8-bit channel value cut to 5 / 6 / 4 bits at its bit position
        // (yuv2rgb.c:806-844), byte-swapped for the big-endian formats -- the fields do not overlap, so the sum swaps as a whole
        const int kind = (p.rgb16 & 7) - 1, fmt = kind >> 1, bgr = kind & 1;                  // fmt 0 565, 1 555, 2 444
        int d8a, d8b, dga, dgb, dba, dbb;                                                      // (dr1, dr2), (dg1, dg2), (db1, db2)
        if (fmt == 2) {
            const int a0 = 0x070B0408, a1 = 0x0D010E02, a2 = 0x0509060A, a3 = 0x0F030C00;      // ff_dither_4x4_16 rows, bytes [0] [1] [2] [3] (output.c:48-53)
            const int r0 = (y & 3) == 0 ? a0 : (y & 3) == 1 ? a1 : (y & 3) == 2 ? a2 : a3, yb = (y & 3) ^ 3, r1 = yb == 0 ? a0 : yb == 1 ? a1 : yb == 2 ? a2 : a3;
            d8a = r0 & 255; d8b = (r0 >> 8) & 255; dga = d8b; dgb = d8a; dba = r1 & 255; dbb = (r1 >> 8) & 255;
        } else {
            const int e = y & 1;                                                               // dither_2x2_8 = { { 6, 2 }, { 0, 4 } }, dither_2x2_4 = { { 1, 3 }, { 2, 0 } } (output.c:38-46)
            d8a = e ? 0 : 6; d8b = e ? 4 : 2; dba = e ? 6 : 0; dbb = e ? 2 : 4;
            if (fmt == 0) { dga = e ? 2 : 1; dgb = e ? 0 : 3; } else { dga = d8b; dgb = d8a; }
        }
        const int rs = fmt == 2 ? 4 : 3, gs = fmt == 0 ? 2 : fmt == 1 ? 3 : 4, gb = fmt == 2 ? 4 : 5, hb = fmt == 0 ? 11 : fmt == 1 ? 10 : 8;
        const int rb = bgr ? 0 : hb, bb = bgr ? hb : 0;
        auto px = [&](int Y, int dr, int dg, int db) -> uint32_t {
            const uint32_t v = (uint32_t)(clip_u8((p.k.cy * (Y + dr) + t.tr) >> 16) >> rs) << rb | (uint32_t)(clip_u8((p.k.cy * (Y + dg) + t.tg) >> 16) >> gs) << gb |
                               (uint32_t)(clip_u8((p.k.cy * (Y + db) + t.tb) >> 16) >> rs) << bb;
            return (p.rgb16 & 8) ? ((v >> 8) | (v << 8)) & 0xffffu : v;
        };
        uint16_t *d16 = reinterpret_cast<uint16_t *>(dst + (size_t)y * dstStride) + 2 * i;
        d16[0] = (uint16_t)px(Y1, d8a, dga, dba);
        if (has2 || dstStride >= 2 * (p.dstW + 1)) d16[1] = (uint16_t)px(Y2, d8b, dgb, dbb);
        return;
    }
    int tr = p.bgr ? t.tb : t.tr, tb = p.bgr ? t.tr : t.tb;
    uint8_t *d = dst + (size_t)y * dstStride + (size_t)i * 6;
    d[0] = (uint8_t)clip_u8((p.k.cy * Y1 + tr) >> 16);
    d[1] = (uint8_t)clip_u8((p.k.cy * Y1 + t.tg) >> 16);
    d[2] = (uint8_t)clip_u8((p.k.cy * Y1 + tb) >> 16);
    if (!has2 && dstStride < 3 * (p.dstW + 1)) return;         // odd width, no room for the pair's second pixel
    d[3] = (uint8_t)clip_u8((p.k.cy * Y2 + tr) >> 16);
    d[4] = (uint8_t)clip_u8((p.k.cy * Y2 + t.tg) >> 16);
    d[5] = (uint8_t)clip_u8((p.k.cy * Y2 + tb) >> 16);
}

// pass 1, four outputs per thread, one 8-byte store (dstW % 4 == 0 not required: the line planes are padded to 8)
__global__ void __launch_bounds__(256)
sws_hscale8to15_x4_kernel(const uint8_t *__restrict__ src, int srcStride, int16_t *__restrict__ dst, int dstStridePx,
                          const int16_t *__restrict__ filter, const int32_t *__restrict__ pos, int fs, int dstW, int rows)
{
    const int i0 = (blockIdx.x * blockDim.x + threadIdx.x) * 4, y = blockIdx.y;
    if (i0 >= dstW || y >= rows) return;
    const uint8_t *srow = src + (size_t)y * srcStride;
    int v[4];
#pragma unroll
    for (int k = 0; k < 4; k++) {
        const int i = min(i0 + k, dstW - 1);
        const uint8_t *sp = srow + pos[i];
        const int16_t *f = filter + (size_t)i * fs;
        int acc = 0;
        for (int j = 0; j < fs; j++) acc += (int)sp[j] * f[j];
        v[k] = i0 + k < dstW ? min(acc >> 7, (1 << 15) - 1) : 0;       // columns past dstW stay zero like the reference's line buffer
    }
    *reinterpret_cast<uint2 *>(dst + (size_t)y * dstStridePx + i0) = make_uint2(pack16(v[0], v[1]), pack16(v[2], v[3]));
}

// pass 2, yuv2rgb24_X_c (output.c:936-995) for 8 pixels per thread: 16-byte luma / 8-byte chroma line loads, three 8-byte stores
__global__ void __launch_bounds__(128)
sws_vscale_rgb24_x8_kernel(SwsDev p, const int16_t *__restrict__ lum, const int16_t *__restrict__ chrU,
                           const int16_t *__restrict__ chrV, int lumStride, int chrStride, uint8_t *__restrict__ dst, int dstStride)
{
    const int gx = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y;
    if (gx * 8 >= p.dstW || y >= p.dstH) return;
    const int fl = p.vLumSize, fc = p.vChrSize;
    const int firstL = max(1 - fl, p.vLumP[y]), firstC = max(1 - fc, p.vChrP[y]);
    const int16_t *lf = p.vLumF + (size_t)y * fl, *cf = p.vChrF + (size_t)y * fc;
    int Y[8], U[4], V[4];
#pragma unroll
    for (int k = 0; k < 8; k++) Y[k] = 1 << 18;
#pragma unroll
    for (int k = 0; k < 4; k++) U[k] = V[k] = 1 << 18;
    for (int j = 0; j < fl; j++) {
        const uint4 w = *reinterpret_cast<const uint4 *>(lum + (size_t)line_index(firstL, j, p.srcH) * lumStride + gx * 8);
        const int c = lf[j];
        Y[0] += lo16s(w.x) * c; Y[1] += hi16s(w.x) * c; Y[2] += lo16s(w.y) * c; Y[3] += hi16s(w.y) * c;
        Y[4] += lo16s(w.z) * c; Y[5] += hi16s(w.z) * c; Y[6] += lo16s(w.w) * c; Y[7] += hi16s(w.w) * c;
    }
    for (int j = 0; j < fc; j++) {
        const size_t o = (size_t)line_index(firstC, j, p.chrSrcH) * chrStride + gx * 4;
        const uint2 wu = *reinterpret_cast<const uint2 *>(chrU + o), wv = *reinterpret_cast<const uint2 *>(chrV + o);
        const int c = cf[j];
        U[0] += lo16s(wu.x) * c; U[1] += hi16s(wu.x) * c; U[2] += lo16s(wu.y) * c; U[3] += hi16s(wu.y) * c;
        V[0] += lo16s(wv.x) * c; V[1] += hi16s(wv.x) * c; V[2] += lo16s(wv.y) * c; V[3] += hi16s(wv.y) * c;
    }
    int r[8], g[8], b[8];
#pragma unroll
    for (int c = 0; c < 4; c++) {
        int y1 = Y[2 * c] >> 19, y2 = Y[2 * c + 1] >> 19, u = U[c] >> 19, v = V[c] >> 19;
        clip_if_flagged(y1, y2, u, v);
        const ChromaTerms t = chroma_terms(u, v, p.k);
        const int tr = p.bgr ? t.tb : t.tr, tb = p.bgr ? t.tr : t.tb;
        r[2 * c] = (p.k.cy * y1 + tr) >> 16; g[2 * c] = (p.k.cy * y1 + t.tg) >> 16; b[2 * c] = (p.k.cy * y1 + tb) >> 16;
        r[2 * c + 1] = (p.k.cy * y2 + tr) >> 16; g[2 * c + 1] = (p.k.cy * y2 + t.tg) >> 16; b[2 * c + 1] = (p.k.cy * y2 + tb) >> 16;
    }
    uint2 *d = reinterpret_cast<uint2 *>(dst + (size_t)y * dstStride + (size_t)gx * 24);
    d[0] = make_uint2(pack4_sat_u8(r[0], g[0], b[0], r[1]), pack4_sat_u8(g[1], b[1], r[2], g[2]));
    d[1] = make_uint2(pack4_sat_u8(b[2], r[3], g[3], b[3]), pack4_sat_u8(r[4], g[4], b[4], r[5]));
    d[2] = make_uint2(pack4_sat_u8(g[5], b[5], r[6], g[6]), pack4_sat_u8(b[6], r[7], g[7], b[7]));
}

// pass 2, SWS_FULL_CHR_H_INT: yuv2rgb24_full_X_c (output.c:1165-1240), thread = (pixel, output row)
__global__ void __launch_bounds__(256)
sws_vscale_rgb24_full_kernel(SwsDev p, const int16_t *__restrict__ lum, const int16_t *__restrict__ chrU,
                             const int16_t *__restrict__ chrV, int lumStride, int chrStride, uint8_t *__restrict__ dst, int dstStride)
{
    const int i = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y;
    if (i >= p.dstW || y >= p.dstH) return;
    const int fl = p.vLumSize, fc = p.vChrSize;
    const int firstL = max(1 - fl, p.vLumP[y]), firstC = max(1 - fc, p.vChrP[y]);
    const int16_t *lf = p.vLumF + (size_t)y * fl, *cf = p.vChrF + (size_t)y * fc;
    int Y = 0, U = -128 * (1 << 19), V = -128 * (1 << 19);
    for (int j = 0; j < fl; j++) Y += lum[(size_t)line_index(firstL, j, p.srcH) * lumStride + i] * lf[j];
    for (int j = 0; j < fc; j++) {
        const size_t o = (size_t)line_index(firstC, j, p.chrSrcH) * chrStride + i;
        U += chrU[o] * cf[j]; V += chrV[o] * cf[j];
    }
    full_pixel(Y >> 10, U >> 10, V >> 10, p.k, p.bgr, dst + (size_t)y * dstStride + (size_t)i * 3);
}

// GENERAL path, pass 1 for 9 / 10 / 16-bit planar sources: hScale16To15_c (swscale.c:110-131): 16-bit words (byte-swapped first for the
// big-endian formats: input.c bswap16Y_c / bswap16UV_c), products shifted down by depth - 1; thread = (column, row)
__global__ void __launch_bounds__(256)
sws_hscale16to15_kernel(const uint8_t *__restrict__ src, int srcStride, int16_t *__restrict__ dst, int dstStridePx,
                        const int16_t *__restrict__ filter, const int32_t *__restrict__ pos, int fs, int dstW, int rows, int bits, int be)
{
    const int i = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y;
    if (i >= dstW || y >= rows) return;
    const uint16_t *s = reinterpret_cast<const uint16_t *>(src + (size_t)y * srcStride) + pos[i];
    const int16_t *f = filter + (size_t)i * fs;
    int val = 0;
    for (int j = 0; j < fs; j++) val += swap16_if(s[j], be) * f[j];
    dst[(size_t)y * dstStridePx + i] = (int16_t)min(val >> (bits - 1), (1 << 15) - 1);
}

// ff_dither_8x8_128[row][col] (swscale.c:38-47) is a bit-interleaved ordered-dither matrix: affine over GF(2) in the bits of row and column
__device__ __forceinline__ int dither128(int row, int col)
{
    int v = 18;
    if (row & 1) v ^= 32;
    if (row & 2) v ^= 8;
    if (row & 4) v ^= 2;
    if (col & 1) v ^= 48;
    if (col & 2) v ^= 12;
    if (col & 4) v ^= 3;
    return 2 * v;
}

// pass 2 for planar output (see plane_store above); dither: 8-bit output of a high-bit-depth source, lumDither8 / chrDither8 with offset doff
__global__ void __launch_bounds__(256)
sws_vscale_plane_kernel(const int16_t *__restrict__ src, int srcStride, int srcH, const int16_t *__restrict__ filter,
                        const int32_t *__restrict__ pos, int fs, uint8_t *__restrict__ dst, int dstStride, int dstW, int dstH, int bits, int be, int step = 1,
                        int dither = 0, int doff = 0)
{
    const int i = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y;
    if (i >= dstW || y >= dstH) return;
    const int first = max(1 - fs, pos[y]);
    int val;
    const int dth = (dither && bits == 8) ? dither128(y & 7, (i + doff) & 7) : 1 << (14 - bits);      // 64 for plain 8-bit output
    if (fs == 1) {
        val = (src[(size_t)line_index(first, 0, srcH) * srcStride + i] + dth) >> (15 - bits);
    } else {
        const int16_t *f = filter + (size_t)y * fs;
        val = bits == 8 ? dth << 12 : 1 << (26 - bits);
        for (int j = 0; j < fs; j++) val += src[(size_t)line_index(first, j, srcH) * srcStride + i] * f[j];
        val >>= 27 - bits;
    }
    plane_store(dst + (size_t)y * dstStride, i * step, plane_clip(val, bits), bits, be);
}

// ---------------------------------------------------------------------------------------------------
// GENERAL path, fused per tile (default): a CTA owns a 128 x 16 tile of the OUTPUT.  It runs hScale8To15 (or the
// fast-bilinear variant) for just the source lines its 16 rows' vertical filters touch, keeps those 15-bit lines in
// shared memory, and runs the vertical filter + output stage from there -- the int16 line planes of the two-pass path
// never exist in HBM.  Same integer recipe as the two-pass kernels above, which stay as the fallback for filters whose
// line window does not fit in shared memory (heavy down-scaling).
// ---------------------------------------------------------------------------------------------------
constexpr int GT_W = 128, GT_H = 16, GT_THREADS = 256;
// a shared luma line: the 8 samples of pixel group g live as two 16-byte quads at words 4g and 80 + 4g, so both the
// column-per-lane stores of the horizontal pass and the two LDS.128 of the vertical pass are bank-conflict free
constexpr int GT_LW = 144;
__host__ __device__ constexpr int gt_lum_slot(int col) { return ((col >> 3) << 2) + (col & 3) + ((col >> 2) & 1) * 80; }

// lines [lo, hi] the vertical filters of output rows y0..y1 read (after line_index()'s clamp)
static inline void tile_line_window(const int32_t *pos, int fs, int y0, int y1, int srcH, int &lo, int &hi)
{
    lo = 0x7fffffff; hi = -1;
    for (int y = y0; y <= y1; y++) {
        int first = pos[y] > 1 - fs ? pos[y] : 1 - fs, a = first, b = first + fs - 1;
        a = a < 0 ? 0 : (a > srcH - 1 ? srcH - 1 : a); b = b < 0 ? 0 : (b > srcH - 1 ? srcH - 1 : b);
        lo = a < lo ? a : lo; hi = b > hi ? b : hi;
    }
}

// one column of a tile: horizontally scaled samples of lines lo + r, r = r0, r0 + rstep, ... < n, into out[r * W]
// (shared lines hold the 15-bit samples as int32 so the vertical pass multiplies them straight from 16-byte loads)
// FS > 0: compile-time tap count with the coefficients in registers; FS == 0: run-time tap count; FS < 0: fast bilinear
// dp2a on (int16 pair) x (unsigned byte pair): .lo takes bytes 0 and 1 of b, .hi bytes 2 and 3; funnel shift right of the pair hi:lo by a multiple of 8
#ifdef AVB_HOSTSIM
inline int sws_dp2a_lo(uint32_t k, uint32_t b, int c) { return c + (int)(int16_t)(k & 0xffff) * (int)(b & 255) + (int)(int16_t)(k >> 16) * (int)((b >> 8) & 255); }
inline int sws_dp2a_hi(uint32_t k, uint32_t b, int c) { return c + (int)(int16_t)(k & 0xffff) * (int)((b >> 16) & 255) + (int)(int16_t)(k >> 16) * (int)(b >> 24); }
inline uint32_t sws_funnel_r(uint32_t lo, uint32_t hi, int s) { return s ? (lo >> s) | (hi << (32 - s)) : lo; }
#else
__device__ __forceinline__ int sws_dp2a_lo(uint32_t k, uint32_t b, int c) { int d; asm("dp2a.lo.s32.u32 %0, %1, %2, %3;" : "=r"(d) : "r"(k), "r"(b), "r"(c)); return d; }
__device__ __forceinline__ int sws_dp2a_hi(uint32_t k, uint32_t b, int c) { int d; asm("dp2a.hi.s32.u32 %0, %1, %2, %3;" : "=r"(d) : "r"(k), "r"(b), "r"(c)); return d; }
__device__ __forceinline__ uint32_t sws_funnel_r(uint32_t lo, uint32_t hi, int s) { return __funnelshift_r(lo, hi, s); }
#endif

template <int FS>
__device__ __forceinline__ void hscale_column(const uint8_t *__restrict__ src, int srcStride, int lo, int n, int r0, int rstep,
                                              int32_t *out, int W_, int x, int dstW, const int16_t *__restrict__ filter,
                                              const int32_t *__restrict__ pos, int fs, int srcW, unsigned xInc, int chroma, int sh = 7)
{   // sh: 7 = hScale8To15_c, 3 = hScale8To19_c (16-bit destinations; swscale.c:62-100)
    if (x >= dstW) { for (int r = r0; r < n; r += rstep) out[r * W_] = 0; return; }     // the reference's zeroed line tail
    const int step = rstep * srcStride;
    if constexpr (FS < 0) {
        const unsigned xpos = (unsigned)x * xInc, xx = xpos >> 16; const int xa = (xpos & 0xFFFF) >> 9;
        const unsigned xx1 = min(xx + 1, (unsigned)srcW - 1);
        const uint8_t *sp = src + (size_t)(lo + r0) * srcStride;
#pragma unroll 2
        for (int r = r0; r < n; r += rstep, sp += step) {
            const int a = sp[xx], b = sp[xx1];
            out[r * W_] = chroma ? a * (xa ^ 127) + b * xa : (a << 7) + (b - a) * xa;
        }
    } else if constexpr (FS == 4) {
        // four taps: the window's bytes arrive as one or two aligned words, a funnel shift lines them up and two dp2a (int16 pair x byte pair)
        // do the sum -- 2 LDG + 3 ALU per sample instead of 4 byte loads + 4 byte merges + 2 dp2a.  A window whose second word would reach past
        // the row's samples (the last columns) and unaligned planes keep the byte loads.
        const int16_t *f = filter + (size_t)x * 4;
        const uint32_t k01 = (uint16_t)f[0] | (uint32_t)(uint16_t)f[1] << 16, k23 = (uint16_t)f[2] | (uint32_t)(uint16_t)f[3] << 16;
        const int ps = pos[x], a0 = ps & ~3, sft = (ps & 3) * 8;
        const bool vec = !(((uintptr_t)src | (uintptr_t)(unsigned)srcStride) & 3) && (sft == 0 || a0 + 8 <= srcW);
        const int lim = (1 << (22 - sh)) - 1;
        if (vec) {
            const uint8_t *sp = src + a0 + (size_t)(lo + r0) * srcStride;
#pragma unroll 4
            for (int r = r0; r < n; r += rstep, sp += step) {
                const uint32_t w0 = *reinterpret_cast<const uint32_t *>(sp), w1 = sft ? *reinterpret_cast<const uint32_t *>(sp + 4) : 0u;
                const uint32_t W = sws_funnel_r(w0, w1, sft);
                out[r * W_] = min(sws_dp2a_hi(k23, W, sws_dp2a_lo(k01, W, 0)) >> sh, lim);
            }
        } else {
            const uint8_t *sp = src + ps + (size_t)(lo + r0) * srcStride;
            for (int r = r0; r < n; r += rstep, sp += step) {
                const uint32_t W = sp[0] | (uint32_t)sp[1] << 8 | (uint32_t)sp[2] << 16 | (uint32_t)sp[3] << 24;
                out[r * W_] = min(sws_dp2a_hi(k23, W, sws_dp2a_lo(k01, W, 0)) >> sh, lim);
            }
        }
    } else if constexpr (FS > 0) {
        int cf[FS > 0 ? FS : 1];
        const int16_t *f = filter + (size_t)x * FS;
#pragma unroll
        for (int j = 0; j < FS; j++) cf[j] = f[j];
        const uint8_t *sp = src + pos[x] + (size_t)(lo + r0) * srcStride;
#pragma unroll 4
        for (int r = r0; r < n; r += rstep, sp += step) {
            int acc = 0;
#pragma unroll
            for (int j = 0; j < FS; j++) acc += (int)sp[j] * cf[j];
            out[r * W_] = min(acc >> sh, (1 << (22 - sh)) - 1);
        }
    } else {
        const int16_t *f = filter + (size_t)x * fs;
        const uint8_t *sp = src + pos[x] + (size_t)(lo + r0) * srcStride;
        for (int r = r0; r < n; r += rstep, sp += step) {
            int acc = 0;
            for (int j = 0; j < fs; j++) acc += (int)sp[j] * f[j];
            out[r * W_] = min(acc >> sh, (1 << (22 - sh)) - 1);
        }
    }
}

struct TileArgs {
    const uint8_t *y, *u, *v; uint8_t *dst0, *dst1, *dst2;
    int yStride, uStride, vStride, dstStride0, dstStride1, dstStride2;
    size_t yFrame, uFrame, vFrame, dstFrame0, dstFrame1, dstFrame2;
    int lumRows, chrRows;           // shared-memory line capacity (host: maximum over all tiles)
    const int2 *lumWin, *chrWin;    // per tile row: (first line, line count) of the vertical filters' window (host table)
    unsigned lumXInc, chrXInc;      // fast bilinear
    int vec;                        // output rows / bases are 8-byte aligned
};

__device__ __forceinline__ void lds8(const int32_t *p, int (&v)[8])
{
    const int4 a = *reinterpret_cast<const int4 *>(p), b = *reinterpret_cast<const int4 *>(p + 80);
    v[0] = a.x; v[1] = a.y; v[2] = a.z; v[3] = a.w; v[4] = b.x; v[5] = b.y; v[6] = b.z; v[7] = b.w;
}
__device__ __forceinline__ void lds4(const int32_t *p, int (&v)[4])
{
    const int4 a = *reinterpret_cast<const int4 *>(p);
    v[0] = a.x; v[1] = a.y; v[2] = a.z; v[3] = a.w;
}

template <int FSL, int FSC, bool FULL = false>
__global__ void __launch_bounds__(GT_THREADS)
sws_tile_rgb24_kernel(SwsDev p, TileArgs a)
{
    extern __shared__ __align__(16) int32_t gt_smem[];
    int32_t *lumS = gt_smem, *chrUS = gt_smem + a.lumRows * GT_LW;
    const int chrPlane = a.chrRows * (FULL ? GT_LW : GT_W / 2);   // V lines follow the U lines
    const int tid = threadIdx.x, x0 = blockIdx.x * GT_W, y0 = blockIdx.y * GT_H, y1 = min(y0 + GT_H, p.dstH) - 1;
    const size_t f = blockIdx.z;
    const int2 lw = a.lumWin[blockIdx.y], cw = a.chrWin[blockIdx.y];
    const int lumLo = lw.x, chrLo = cw.x;
    {   // horizontal pass into shared memory
        const int col = tid & (GT_W - 1);
        hscale_column<FSL>(a.y + f * a.yFrame, a.yStride, lumLo, lw.y, tid >> 7, 2, lumS + gt_lum_slot(col), GT_LW, x0 + col, p.dstW,
                           p.hLumF, p.hLumP, p.hLumSize, p.srcW, a.lumXInc, 0);
        const int plane = tid >> 7;
        if (FULL) {                      // one chroma sample per pixel: each plane is as wide as the luma tile, same quad layout
            hscale_column<FSC>((plane ? a.v + f * a.vFrame : a.u + f * a.uFrame), plane ? a.vStride : a.uStride, chrLo, cw.y, 0, 1,
                               chrUS + plane * chrPlane + gt_lum_slot(col), GT_LW, x0 + col, p.chrDstW,
                               p.hChrF, p.hChrP, p.hChrSize, p.chrSrcW, a.chrXInc, 1);
        } else {
            const int ccol = tid & (GT_W / 2 - 1);
            hscale_column<FSC>((plane ? a.v + f * a.vFrame : a.u + f * a.uFrame), plane ? a.vStride : a.uStride, chrLo, cw.y,
                               (tid >> 6) & 1, 2, chrUS + plane * chrPlane + ccol, GT_W / 2, (x0 >> 1) + ccol, p.chrDstW,
                               p.hChrF, p.hChrP, p.hChrSize, p.chrSrcW, a.chrXInc, 1);
        }
    }
    __syncthreads();
    const int tx = tid & 15, y = y0 + (tid >> 4), x = x0 + 8 * tx;
    if (y > y1 || x >= p.dstW) return;
    const int fl = p.vLumSize, fc = p.vChrSize;
    const int firstL = max(1 - fl, p.vLumP[y]), firstC = max(1 - fc, p.vChrP[y]);
    const int32_t *lumT = lumS + 4 * tx - lumLo * GT_LW, *chrT = chrUS + 4 * tx - chrLo * (GT_W / 2);
    auto LL = [&](int j) { return lumT + line_index(firstL, j, p.srcH) * GT_LW; };
    if (FULL) {                                                // yuv2rgb24_full_X_c, output.c:1165-1240
        const int16_t *lf = p.vLumF + (size_t)y * fl, *cf = p.vChrF + (size_t)y * fc;
        const int32_t *chrF = chrUS + 4 * tx - chrLo * GT_LW;
        int Y[8], U[8], V[8], t8[8];
#pragma unroll
        for (int k = 0; k < 8; k++) { Y[k] = 0; U[k] = V[k] = -128 * (1 << 19); }
        for (int j = 0; j < fl; j++) {
            lds8(LL(j), t8); const int c = lf[j];
#pragma unroll
            for (int k = 0; k < 8; k++) Y[k] += t8[k] * c;
        }
        for (int j = 0; j < fc; j++) {
            const int c = cf[j]; const int32_t *cl = chrF + line_index(firstC, j, p.chrSrcH) * GT_LW;
            lds8(cl, t8);
#pragma unroll
            for (int k = 0; k < 8; k++) U[k] += t8[k] * c;
            lds8(cl + chrPlane, t8);
#pragma unroll
            for (int k = 0; k < 8; k++) V[k] += t8[k] * c;
        }
        uint8_t *d = a.dst0 + f * a.dstFrame0 + (size_t)y * a.dstStride0 + (size_t)x * 3;
#pragma unroll
        for (int k = 0; k < 8; k++) if (x + k < p.dstW) full_pixel(Y[k] >> 10, U[k] >> 10, V[k] >> 10, p.k, p.bgr, d + 3 * k);
        return;
    }
    auto CC = [&](int j) { return chrT + line_index(firstC, j, p.chrSrcH) * (GT_W / 2); };
    int Y[8], U[4], V[4], t8[8], t4[4];
    if (fl == 1 && fc <= 2) {                                  // yuv2rgb24_1_c, output.c:1042-1110
        const int uvalpha = fc == 1 ? 0 : p.vChrF[2 * y + 1];
        lds8(LL(0), Y);
#pragma unroll
        for (int k = 0; k < 8; k++) Y[k] = clip_u8(Y[k] >> 7);
        const int32_t *c0 = CC(0);
        lds4(c0, U); lds4(c0 + chrPlane, V);
        if (uvalpha < 2048) {
#pragma unroll
            for (int k = 0; k < 4; k++) { U[k] = clip_u8(U[k] >> 7); V[k] = clip_u8(V[k] >> 7); }
        } else {
            const int32_t *c1 = CC(1);
            lds4(c1, t4);
#pragma unroll
            for (int k = 0; k < 4; k++) U[k] = clip_u8((U[k] + t4[k]) >> 8);
            lds4(c1 + chrPlane, t4);
#pragma unroll
            for (int k = 0; k < 4; k++) V[k] = clip_u8((V[k] + t4[k]) >> 8);
        }
    } else if (fl == 2 && fc == 2) {                           // yuv2rgb24_2_c, output.c:997-1040
        const int ya = p.vLumF[2 * y + 1], ua = p.vChrF[2 * y + 1], ya1 = 4096 - ya, ua1 = 4096 - ua;
        lds8(LL(0), Y); lds8(LL(1), t8);
#pragma unroll
        for (int k = 0; k < 8; k++) Y[k] = clip_u8((Y[k] * ya1 + t8[k] * ya) >> 19);
        const int32_t *c0 = CC(0), *c1 = CC(1);
        lds4(c0, U); lds4(c1, t4);
#pragma unroll
        for (int k = 0; k < 4; k++) U[k] = clip_u8((U[k] * ua1 + t4[k] * ua) >> 19);
        lds4(c0 + chrPlane, V); lds4(c1 + chrPlane, t4);
#pragma unroll
        for (int k = 0; k < 4; k++) V[k] = clip_u8((V[k] * ua1 + t4[k] * ua) >> 19);
    } else {                                                   // yuv2rgb24_X_c, output.c:936-995
        const int16_t *lf = p.vLumF + (size_t)y * fl, *cf = p.vChrF + (size_t)y * fc;
#pragma unroll
        for (int k = 0; k < 8; k++) Y[k] = 1 << 18;
#pragma unroll
        for (int k = 0; k < 4; k++) U[k] = V[k] = 1 << 18;
        if (fl == 4 && fc == 4) {                              // bicubic's window: straight-line code, no loop control between the taps
            int lc[4], cc[4];
#pragma unroll
            for (int j = 0; j < 4; j++) { lc[j] = lf[j]; cc[j] = cf[j]; }
#pragma unroll
            for (int j = 0; j < 4; j++) {
                lds8(LL(j), t8);
#pragma unroll
                for (int k = 0; k < 8; k++) Y[k] += t8[k] * lc[j];
            }
#pragma unroll
            for (int j = 0; j < 4; j++) {
                const int32_t *cl = CC(j);
                lds4(cl, t4);
#pragma unroll
                for (int k = 0; k < 4; k++) U[k] += t4[k] * cc[j];
                lds4(cl + chrPlane, t4);
#pragma unroll
                for (int k = 0; k < 4; k++) V[k] += t4[k] * cc[j];
            }
        } else {
#pragma unroll 4
            for (int j = 0; j < fl; j++) {
                lds8(LL(j), t8); const int c = lf[j];
#pragma unroll
                for (int k = 0; k < 8; k++) Y[k] += t8[k] * c;
            }
#pragma unroll 4
            for (int j = 0; j < fc; j++) {
                const int c = cf[j]; const int32_t *cl = CC(j);
                lds4(cl, t4);
#pragma unroll
                for (int k = 0; k < 4; k++) U[k] += t4[k] * c;
                lds4(cl + chrPlane, t4);
#pragma unroll
                for (int k = 0; k < 4; k++) V[k] += t4[k] * c;
            }
        }
#pragma unroll
        for (int k = 0; k < 4; k++) {
            Y[2 * k] >>= 19; Y[2 * k + 1] >>= 19; U[k] >>= 19; V[k] >>= 19;
            clip_if_flagged(Y[2 * k], Y[2 * k + 1], U[k], V[k]);
        }
    }
    int r[8], g[8], b[8];
#pragma unroll
    for (int c = 0; c < 4; c++) {
        const ChromaTerms t = chroma_terms(U[c], V[c], p.k);
        const int tr = p.bgr ? t.tb : t.tr, tb = p.bgr ? t.tr : t.tb;
#pragma unroll
        for (int e = 0; e < 2; e++) {
            const int yy = p.k.cy * Y[2 * c + e];
            r[2 * c + e] = (yy + tr) >> 16; g[2 * c + e] = (yy + t.tg) >> 16; b[2 * c + e] = (yy + tb) >> 16;
        }
    }
    uint8_t *d = a.dst0 + f * a.dstFrame0 + (size_t)y * a.dstStride0 + (size_t)x * 3;
    if (a.vec && x + 8 <= p.dstW) {
        uint2 *dv = reinterpret_cast<uint2 *>(d);
        dv[0] = make_uint2(pack4_sat_u8(r[0], g[0], b[0], r[1]), pack4_sat_u8(g[1], b[1], r[2], g[2]));
        dv[1] = make_uint2(pack4_sat_u8(b[2], r[3], g[3], b[3]), pack4_sat_u8(r[4], g[4], b[4], r[5]));
        dv[2] = make_uint2(pack4_sat_u8(g[5], b[5], r[6], g[6]), pack4_sat_u8(b[6], r[7], g[7], b[7]));
    } else {
        // the C code writes whole pairs: an odd width's last pair spills one pixel into the row padding when there is room
        const int wlim = (p.dstW & 1) && a.dstStride0 >= 3 * (p.dstW + 1) ? p.dstW + 1 : p.dstW;
#pragma unroll
        for (int k = 0; k < 8; k++)
            if (x + k < wlim) { d[3 * k] = (uint8_t)clip_u8(r[k]); d[3 * k + 1] = (uint8_t)clip_u8(g[k]); d[3 * k + 2] = (uint8_t)clip_u8(b[k]); }
    }
}

// planar 8-bit output (yuv2planeX_8_c / yuv2plane1_8_c, output.c:242-265): the same tile scheme for one plane kind;
// CHROMA: blockIdx.z = 2 * frame + plane
template <int FS, bool CHROMA>
__global__ void __launch_bounds__(GT_THREADS)
sws_tile_plane_kernel(SwsDev p, TileArgs a)
{
    extern __shared__ __align__(16) int32_t gt_smem[];
    const int tid = threadIdx.x, x0 = blockIdx.x * GT_W, y0 = blockIdx.y * GT_H;
    const int dstW = CHROMA ? p.chrDstW : p.dstW, dstH = CHROMA ? p.chrDstH : p.dstH, srcH = CHROMA ? p.chrSrcH : p.srcH;
    const int y1 = min(y0 + GT_H, dstH) - 1;
    const size_t f = CHROMA ? blockIdx.z >> 1 : blockIdx.z; const int plane = CHROMA ? 1 + (blockIdx.z & 1) : 0;
    const uint8_t *src = plane == 0 ? a.y + f * a.yFrame : plane == 1 ? a.u + f * a.uFrame : a.v + f * a.vFrame;
    const int srcStride = plane == 0 ? a.yStride : plane == 1 ? a.uStride : a.vStride;
    uint8_t *dst = plane == 0 ? a.dst0 + f * a.dstFrame0 : plane == 1 ? a.dst1 + f * a.dstFrame1 : a.dst2 + f * a.dstFrame2;
    const int dstStride = plane == 0 ? a.dstStride0 : plane == 1 ? a.dstStride1 : a.dstStride2;
    const int16_t *vF = CHROMA ? p.vChrF : p.vLumF; const int32_t *vP = CHROMA ? p.vChrP : p.vLumP;
    const int fs = CHROMA ? p.vChrSize : p.vLumSize;
    const int2 win = (CHROMA ? a.chrWin : a.lumWin)[blockIdx.y];
    const int lo = win.x;
    {
        const int col = tid & (GT_W - 1);
        hscale_column<FS>(src, srcStride, lo, win.y, tid >> 7, 2, gt_smem + gt_lum_slot(col), GT_LW, x0 + col, dstW,
                          CHROMA ? p.hChrF : p.hLumF, CHROMA ? p.hChrP : p.hLumP, CHROMA ? p.hChrSize : p.hLumSize,
                          CHROMA ? p.chrSrcW : p.srcW, CHROMA ? a.chrXInc : a.lumXInc, CHROMA, p.dstBits == 16 ? 3 : 7);
    }
    __syncthreads();
    const int tx = tid & 15, y = y0 + (tid >> 4), x = x0 + 8 * tx;
    if (y > y1 || x >= dstW) return;
    const int first = max(1 - fs, vP[y]);
    int v[8], t8[8];
    const int bits = p.dstBits;
    if (bits == 16) {            // yuv2plane1_16_c / yuv2planeX_16_c (output.c:136-172) on the 19-bit lines
        if (fs == 1) {
            lds8(gt_smem + (line_index(first, 0, srcH) - lo) * GT_LW + 4 * tx, v);
#pragma unroll
            for (int k = 0; k < 8; k++) v[k] = min(max((v[k] + 4) >> 3, 0), 65535);
        } else {
            const int16_t *cf = vF + (size_t)y * fs;
            unsigned acc[8];      // the reference biases the sum by -0x40000000 so it stays inside 32 bits; wrap-around arithmetic here
#pragma unroll
            for (int k = 0; k < 8; k++) acc[k] = (1u << 14) - 0x40000000u;
            for (int j = 0; j < fs; j++) {
                lds8(gt_smem + (line_index(first, j, srcH) - lo) * GT_LW + 4 * tx, t8); const int c = cf[j];
#pragma unroll
                for (int k = 0; k < 8; k++) acc[k] += (unsigned)(t8[k] * c);
            }
#pragma unroll
            for (int k = 0; k < 8; k++) v[k] = min(max((int)acc[k] >> 15, -32768), 32767) + 0x8000;
        }
#pragma unroll
        for (int k = 0; k < 8; k++) v[k] = swap16_if(v[k], p.dstBE);
        uint16_t *d16 = reinterpret_cast<uint16_t *>(dst + (size_t)y * dstStride) + x;
        if (x + 8 <= dstW && !(((uintptr_t)d16) & 15))
            *reinterpret_cast<uint4 *>(d16) = make_uint4(v[0] | (v[1] << 16), v[2] | (v[3] << 16), v[4] | (v[5] << 16), v[6] | (v[7] << 16));
        else
#pragma unroll
            for (int k = 0; k < 8; k++) if (x + k < dstW) d16[k] = (uint16_t)v[k];
        return;
    }
    if (fs == 1) {
        lds8(gt_smem + (line_index(first, 0, srcH) - lo) * GT_LW + 4 * tx, v);
#pragma unroll
        for (int k = 0; k < 8; k++) v[k] = (v[k] + (1 << (14 - bits))) >> (15 - bits);
    } else {
        const int16_t *cf = vF + (size_t)y * fs;
#pragma unroll
        for (int k = 0; k < 8; k++) v[k] = 1 << (26 - bits);
        for (int j = 0; j < fs; j++) {
            lds8(gt_smem + (line_index(first, j, srcH) - lo) * GT_LW + 4 * tx, t8); const int c = cf[j];
#pragma unroll
            for (int k = 0; k < 8; k++) v[k] += t8[k] * c;
        }
#pragma unroll
        for (int k = 0; k < 8; k++) v[k] >>= 27 - bits;
    }
    if (bits != 8) {
        uint16_t *d16 = reinterpret_cast<uint16_t *>(dst + (size_t)y * dstStride) + x;
#pragma unroll
        for (int k = 0; k < 8; k++) v[k] = swap16_if(plane_clip(v[k], bits), p.dstBE);
        if (x + 8 <= dstW && !(((uintptr_t)d16) & 15))
            *reinterpret_cast<uint4 *>(d16) = make_uint4(v[0] | (v[1] << 16), v[2] | (v[3] << 16), v[4] | (v[5] << 16), v[6] | (v[7] << 16));
        else
#pragma unroll
            for (int k = 0; k < 8; k++) if (x + k < dstW) d16[k] = (uint16_t)v[k];
        return;
    }
    if (CHROMA && p.chrStep == 2) {          // nv12 / nv21: this plane's samples go to every other byte
        uint8_t *d2 = dst + (size_t)y * dstStride + 2 * x;
#pragma unroll
        for (int k = 0; k < 8; k++) if (x + k < dstW) d2[2 * k] = (uint8_t)clip_u8(v[k]);
        return;
    }
    uint8_t *d = dst + (size_t)y * dstStride + x;
    if (x + 8 <= dstW && !(((uintptr_t)d) & 7)) {
        *reinterpret_cast<uint2 *>(d) = make_uint2(pack4_sat_u8(v[0], v[1], v[2], v[3]), pack4_sat_u8(v[4], v[5], v[6], v[7]));
    } else {
#pragma unroll
        for (int k = 0; k < 8; k++) if (x + k < dstW) d[k] = (uint8_t)clip_u8(v[k]);
    }
}

// nv12ToUV_c / nv21ToUV_c (input.c:475-497) for whole planes: one thread splits 4 (U,V) pairs
__global__ void __launch_bounds__(256)
sws_split_nv_kernel(const uint8_t *__restrict__ uv, int uvStride, size_t uvFrame, uint8_t *__restrict__ u, uint8_t *__restrict__ v,
                    int outStride, size_t outFrameU, size_t outFrameV, int w, int h)
{
    const int x4 = (blockIdx.x * blockDim.x + threadIdx.x) * 4, y = blockIdx.y;
    if (x4 >= w || y >= h) return;
    const size_t f = blockIdx.z;
    const uint8_t *s = uv + f * uvFrame + (size_t)y * uvStride + 2 * x4;
    uint8_t *du = u + f * outFrameU + (size_t)y * outStride + x4, *dv = v + f * outFrameV + (size_t)y * outStride + x4;
    if (x4 + 4 <= w && !(((uintptr_t)s) & 7) && !(((uintptr_t)du | (uintptr_t)dv) & 3)) {
        const uint2 p = *reinterpret_cast<const uint2 *>(s);
        *reinterpret_cast<uint32_t *>(du) = __byte_perm(p.x, p.y, 0x6420);
        *reinterpret_cast<uint32_t *>(dv) = __byte_perm(p.x, p.y, 0x7531);
    } else {
        for (int k = 0; k < 4 && x4 + k < w; k++) { du[k] = s[2 * k]; dv[k] = s[2 * k + 1]; }
    }
}

// ---------------------------------------------------------------------------------------------------
// packed sources: the reference's input readers (lumToYV12 / chrToYV12, libswscale/input.c) for whole frames, in front of
// the planar kernels.  The readers run on 8-bit samples and produce 8-bit planes (formatConvBuffer, swscale.c:120-160).
// ---------------------------------------------------------------------------------------------------
namespace rd {            // input.c:38-47
constexpr int SH = 15;
constexpr int BY = (int)(0.114 * 219 / 255 * (1 << SH) + 0.5), BV = -(int)(0.081 * 224 / 255 * (1 << SH) + 0.5), BU = (int)(0.500 * 224 / 255 * (1 << SH) + 0.5);
constexpr int GY = (int)(0.587 * 219 / 255 * (1 << SH) + 0.5), GV = -(int)(0.419 * 224 / 255 * (1 << SH) + 0.5), GU = -(int)(0.331 * 224 / 255 * (1 << SH) + 0.5);
constexpr int RY = (int)(0.299 * 219 / 255 * (1 << SH) + 0.5), RV = (int)(0.500 * 224 / 255 * (1 << SH) + 0.5), RU = -(int)(0.169 * 224 / 255 * (1 << SH) + 0.5);
}

// KIND 1: rgb24 / bgr24 (rgb24ToY_c, rgb24ToUV_c, rgb24ToUV_half_c and the bgr24 twins, input.c:539-625; `ro` / `go` / `bo` are the byte
// offsets of red, green and blue), KIND 4: argb / rgba / abgr / bgra (the rgb16_32ToY / ToUV / ToUV_half templates, input.c:230-330:
// the same sums on the 8-bit channels, scaled by 2^8 on both sides of the shift), 2: yuyv422 (yuy2ToY_c, yuy2ToUV_c, :369-387), 3: uyvy422 (uyvyToY_c, uyvyToUV_c, :456-473).
// One thread reads one pixel pair.  For an odd width the reference's chroma readers read one pixel past the row; those bytes
// are read here too whenever they lie inside the frame (row padding or the next row), else the pair's first pixel is repeated.
template <int KIND>
__global__ void __launch_bounds__(256)
sws_read_packed_kernel(const uint8_t *__restrict__ src, int srcStride, size_t srcFrame, uint8_t *__restrict__ Y, uint8_t *__restrict__ U,
                       uint8_t *__restrict__ V, int yPitch, int cPitch, size_t yPlane, size_t cPlane, int w, int h, int ro, int go, int bo, int half)
{
    const int i = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y;
    if (2 * i >= w) return;
    const size_t f = blockIdx.z;
    constexpr int BPP = KIND == 1 ? 3 : KIND == 4 ? 4 : 2;
    const uint8_t *s = src + f * srcFrame + (size_t)y * srcStride + (size_t)i * 2 * BPP;
    uint8_t *dy = Y + f * yPlane + (size_t)y * yPitch + 2 * i;
    uint8_t *du = U + f * cPlane + (size_t)y * cPitch, *dv = V + f * cPlane + (size_t)y * cPitch;
    const bool second = 2 * i + 1 < w;
    const bool readable = second || y < h - 1 || (2 * i + 2) * BPP <= srcStride;
    if (KIND == 1 || KIND == 4) {
        using namespace rd;
        const int r0 = s[ro], g0 = s[go], b0 = s[bo];
        int r1 = r0, g1 = g0, b1 = b0;
        if (readable) { r1 = s[BPP + ro]; g1 = s[BPP + go]; b1 = s[BPP + bo]; }
        dy[0] = (uint8_t)((RY * r0 + GY * g0 + BY * b0 + (33 << (SH - 1))) >> SH);
        if (second) dy[1] = (uint8_t)((RY * r1 + GY * g1 + BY * b1 + (33 << (SH - 1))) >> SH);
        if (half) {
            const int r = r0 + r1, g = g0 + g1, b = b0 + b1;
            du[i] = (uint8_t)((RU * r + GU * g + BU * b + (257 << SH)) >> (SH + 1));
            dv[i] = (uint8_t)((RV * r + GV * g + BV * b + (257 << SH)) >> (SH + 1));
        } else {
            du[2 * i] = (uint8_t)((RU * r0 + GU * g0 + BU * b0 + (257 << (SH - 1))) >> SH);
            dv[2 * i] = (uint8_t)((RV * r0 + GV * g0 + BV * b0 + (257 << (SH - 1))) >> SH);
            if (second) {
                du[2 * i + 1] = (uint8_t)((RU * r1 + GU * g1 + BU * b1 + (257 << (SH - 1))) >> SH);
                dv[2 * i + 1] = (uint8_t)((RV * r1 + GV * g1 + BV * b1 + (257 << (SH - 1))) >> SH);
            }
        }
    } else {
        const int yo = KIND == 2 ? 0 : 1, co = KIND == 2 ? 1 : 0;
        dy[0] = s[yo];
        if (second) dy[1] = s[2 + yo];
        du[i] = s[co];
        dv[i] = readable ? s[2 + co] : s[co];
    }
}

// pal8 sources: src = one index per pixel, pal = 256 native-endian 0xAARRGGBB words (per frame).  sws_scale() converts the palette to limited-range
// y / u / v for every call (swscale_unscaled.c:1236-1268, constants of swscale_internal.h with RGB2YUV_SHIFT 15, av_clip_uint8 on each) and the readers
// palToY_c / palToUV_c look the samples up (input.c:321-343) -- chroma at full resolution.  Here a thread converts its own pixel's entry.
__device__ __forceinline__ void pal8_entry(const uint32_t *__restrict__ pal, int i, int &r, int &g, int &b)
{
    const uint32_t p = pal[i];
    r = (p >> 16) & 255; g = (p >> 8) & 255; b = p & 255;
}
__global__ void __launch_bounds__(256)
sws_read_pal8_kernel(const uint8_t *__restrict__ src, int srcStride, size_t srcFrame, const uint8_t *__restrict__ pal, size_t palFrame, uint8_t *__restrict__ Y,
                     uint8_t *__restrict__ U, uint8_t *__restrict__ V, int pitch, size_t plane, int w, int h)
{
    const int x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y;
    if (x >= w) return;
    const size_t f = blockIdx.z;
    using namespace rd;
    int r, g, b;
    pal8_entry(reinterpret_cast<const uint32_t *>(pal + f * palFrame), src[f * srcFrame + (size_t)y * srcStride + x], r, g, b);
    const size_t o = f * plane + (size_t)y * pitch + x;
    Y[o] = (uint8_t)clip_u8((RY * r + GY * g + BY * b + (33 << (SH - 1))) >> SH);
    U[o] = (uint8_t)clip_u8((RU * r + GU * g + BU * b + (257 << (SH - 1))) >> SH);
    V[o] = (uint8_t)clip_u8((RV * r + GV * g + BV * b + (257 << (SH - 1))) >> SH);
}
// palToRgbWrapper (swscale_unscaled.c:342-384): same size to 24 / 32-bit rgb is a palette lookup, alpha 255 (the table of :1270-1295); map as in
// sws_rgb_map_kernel with source "bytes" 0 = r, 1 = g, 2 = b
__global__ void __launch_bounds__(256)
sws_pal8_rgb_kernel(const uint8_t *__restrict__ src, int srcStride, size_t srcFrame, const uint8_t *__restrict__ pal, size_t palFrame, uint8_t *__restrict__ dst,
                    int dstStride, size_t dstFrame, int w, int h, int dbpp, unsigned map)
{
    const int x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y;
    if (x >= w) return;
    const size_t f = blockIdx.z;
    int v[3];
    pal8_entry(reinterpret_cast<const uint32_t *>(pal + f * palFrame), src[f * srcFrame + (size_t)y * srcStride + x], v[0], v[1], v[2]);
    uint8_t *d = dst + f * dstFrame + (size_t)y * dstStride + (size_t)dbpp * x;
    for (int k = 0; k < dbpp; k++) { const unsigned m = (map >> (4 * k)) & 15; d[k] = m == 15 ? (uint8_t)255 : (uint8_t)v[m]; }
}

// the reference's unscaled special converters for these sources (swscale_unscaled.c:1063-1072,1140-1145):
// rgb24 <-> bgr24 (rgbToRgbWrapper -> rgb24tobgr24, rgb2rgb_template.c) and the same-format copy (packedCopyWrapper); only the
// w x h pixels are written (the reference's whole-buffer variants also convert the row padding when the strides match)
__global__ void __launch_bounds__(256)
sws_rgb24_shuffle_kernel(const uint8_t *__restrict__ src, int srcStride, size_t srcFrame, uint8_t *__restrict__ dst, int dstStride, size_t dstFrame,
                         int w, int h, int swap)
{
    const int x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y;
    if (x >= w) return;
    const uint8_t *s = src + blockIdx.z * srcFrame + (size_t)y * srcStride + 3 * x;
    uint8_t *d = dst + blockIdx.z * dstFrame + (size_t)y * dstStride + 3 * x;
    const uint8_t a = s[0], b = s[1], c = s[2];
    d[0] = swap ? c : a; d[1] = b; d[2] = swap ? a : c;
}

// rgbToRgbWrapper's 24 <-> 32 and 32 <-> 32 bit byte converters (rgb2rgb.c:139-175,335-352, rgb2rgb_template.c:31-78,338-350; choice at
// swscale_unscaled.c:590-660): each is a channel remap -- alpha copied 32 -> 32, 255 for 24 -> 32, dropped 32 -> 24.  map = four nibbles, nibble k =
// the source byte stored to destination byte k (15: the constant 255).  One thread per pixel.
__global__ void __launch_bounds__(256)
sws_rgb_map_kernel(const uint8_t *__restrict__ src, int srcStride, size_t srcFrame, uint8_t *__restrict__ dst, int dstStride, size_t dstFrame,
                   int w, int h, int sbpp, int dbpp, unsigned map)
{
    const int x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y;
    if (x >= w) return;
    const uint8_t *s = src + blockIdx.z * srcFrame + (size_t)y * srcStride + (size_t)sbpp * x;
    uint8_t *d = dst + blockIdx.z * dstFrame + (size_t)y * dstStride + (size_t)dbpp * x;
    uint8_t v[4];
    for (int k = 0; k < sbpp; k++) v[k] = s[k];
    for (int k = 0; k < dbpp; k++) { const unsigned m = (map >> (4 * k)) & 15; d[k] = m == 15 ? (uint8_t)255 : v[m]; }
}

// bgr24ToYv12Wrapper -> rgb24toyv12_c (rgb2rgb_template.c:638-693, 8-bit coefficients rgb2rgb.c:111-120): chroma from the first
// pixel of each pair of the even rows only; width >> 1 pairs, so an odd last column stays untouched.  One thread per pair and row.
__global__ void __launch_bounds__(256)
sws_bgr24_yv12_kernel(const uint8_t *__restrict__ src, int srcStride, size_t srcFrame, uint8_t *__restrict__ Y, uint8_t *__restrict__ U,
                      uint8_t *__restrict__ V, int yStride, int cStride, size_t yFrame, size_t uFrame, size_t vFrame, int w, int h)
{
    const int i = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y;
    if (i >= (w >> 1)) return;
    const size_t f = blockIdx.z;
    const uint8_t *s = src + f * srcFrame + (size_t)y * srcStride + 6 * i;
    uint8_t *dy = Y + f * yFrame + (size_t)y * yStride + 2 * i;
    const int b0 = s[0], g0 = s[1], r0 = s[2], b1 = s[3], g1 = s[4], r1 = s[5];
    dy[0] = (uint8_t)(((66 * r0 + 129 * g0 + 25 * b0) >> 8) + 16);
    dy[1] = (uint8_t)(((66 * r1 + 129 * g1 + 25 * b1) >> 8) + 16);
    if (!(y & 1)) {
        U[f * uFrame + (size_t)(y >> 1) * cStride + i] = (uint8_t)(((-37 * r0 - 73 * g0 + 112 * b0) >> 8) + 128);
        V[f * vFrame + (size_t)(y >> 1) * cStride + i] = (uint8_t)(((112 * r0 - 93 * g0 - 17 * b0) >> 8) + 128);
    }
}

// yuyvToYuv420Wrapper / uyvyToYuv420Wrapper -> yuyvtoyuv420_c / uyvytoyuv420_c (rgb2rgb_template.c:854-910): luma of every row,
// chroma = the mean (truncating) of the two rows of a pair; h / 2 chroma rows.  One thread per pixel pair and row.
__global__ void __launch_bounds__(256)
sws_yuyv_yv12_kernel(const uint8_t *__restrict__ src, int srcStride, size_t srcFrame, uint8_t *__restrict__ Y, uint8_t *__restrict__ U,
                     uint8_t *__restrict__ V, int yStride, int cStride, size_t yFrame, size_t uFrame, size_t vFrame, int w, int h, int uyvy)
{
    const int i = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y;
    if (2 * i >= w) return;
    const size_t f = blockIdx.z;
    const uint8_t *s = src + f * srcFrame + (size_t)y * srcStride + 4 * i;
    uint8_t *dy = Y + f * yFrame + (size_t)y * yStride + 2 * i;
    const int yo = uyvy ? 1 : 0, co = uyvy ? 0 : 1;
    const bool second = 2 * i + 1 < w;
    dy[0] = s[yo];
    if (second) dy[1] = s[2 + yo];
    if (y & 1) {
        const uint8_t *p = s - srcStride;
        // the V sample one pixel past an odd width lies in the row padding or in the next row (the reference reads it too)
        const int v0 = p[2 + co], v1 = (second || 4 * i + 4 <= srcStride || y < h - 1) ? s[2 + co] : s[co];
        U[f * uFrame + (size_t)(y >> 1) * cStride + i] = (uint8_t)((p[co] + s[co]) >> 1);
        V[f * vFrame + (size_t)(y >> 1) * cStride + i] = (uint8_t)((v0 + v1) >> 1);
    }
}

// 32-bit packed rgb destinations (argb, rgba, abgr, bgra): the colour tables of the 32-bit output functions hold the same 8-bit
// channel values as the 24-bit ones plus a constant alpha of 255 (yuv2rgb.c:763-800, output.c:1040-1075,1230-1260), so the rgb24
// result is expanded: `ro` / `go` / `bo` / `ao` are the byte positions inside a destination pixel.  One thread per pixel.
__global__ void __launch_bounds__(256)
sws_expand_rgb32_kernel(const uint8_t *__restrict__ src, int srcStride, size_t srcFrame, uint8_t *__restrict__ dst, int dstStride, size_t dstFrame,
                        int w, int ro, int go, int bo, int ao)
{
    const int x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y;
    if (x >= w) return;
    const uint8_t *s = src + blockIdx.z * srcFrame + (size_t)y * srcStride + 3 * x;
    const uint32_t v = ((uint32_t)s[0] << (8 * ro)) | ((uint32_t)s[1] << (8 * go)) | ((uint32_t)s[2] << (8 * bo)) | (255u << (8 * ao));
    uint8_t *d = dst + blockIdx.z * dstFrame + (size_t)y * dstStride + 4 * x;
    if (!((uintptr_t)d & 3)) *reinterpret_cast<uint32_t *>(d) = v;
    else { d[0] = (uint8_t)v; d[1] = (uint8_t)(v >> 8); d[2] = (uint8_t)(v >> 16); d[3] = (uint8_t)(v >> 24); }
}

// yuv422pToYuy2Wrapper / yuv422pToUyvyWrapper and planarToYuy2Wrapper / planarToUyvyWrapper (swscale_unscaled.c:183-225 ->
// yuvPlanartoyuy2_c / yuvPlanartouyvy_c, rgb2rgb_template.c:322-420): width >> 1 pixel pairs per row, luma row y with chroma row y >> vshift
__global__ void __launch_bounds__(256)
sws_planar_to_422_kernel(const uint8_t *__restrict__ Y, int yStride, size_t yFrame, const uint8_t *__restrict__ U, const uint8_t *__restrict__ V,
                         int cStride, size_t uFrame, size_t vFrame, uint8_t *__restrict__ dst, int dstStride, size_t dstFrame, int w, int vshift, int uyvy)
{
    const int i = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y;
    if (i >= (w >> 1)) return;
    const size_t f = blockIdx.z;
    const uint8_t *py = Y + f * yFrame + (size_t)y * yStride + 2 * i;
    const uint8_t u = U[f * uFrame + (size_t)(y >> vshift) * cStride + i], v = V[f * vFrame + (size_t)(y >> vshift) * cStride + i];
    uint8_t *d = dst + f * dstFrame + (size_t)y * dstStride + 4 * i;
    if (uyvy) { d[0] = u; d[1] = py[0]; d[2] = v; d[3] = py[1]; } else { d[0] = py[0]; d[1] = u; d[2] = py[1]; d[3] = v; }
}

// planarToNv12Wrapper (swscale_unscaled.c:138-156): interleaveBytes of srcW / 2 x srcH / 2 chroma samples (an odd last column / row stays untouched)
__global__ void __launch_bounds__(256)
sws_interleave_kernel(const uint8_t *__restrict__ a, int aStride, size_t aFrame, const uint8_t *__restrict__ b, int bStride, size_t bFrame,
                      uint8_t *__restrict__ dst, int dstStride, size_t dstFrame, int w)
{
    const int x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y;
    if (x >= w) return;
    uint8_t *d = dst + blockIdx.z * dstFrame + (size_t)y * dstStride + 2 * x;
    d[0] = a[blockIdx.z * aFrame + (size_t)y * aStride + x];
    d[1] = b[blockIdx.z * bFrame + (size_t)y * bStride + x];
}

// planarCopyWrapper, 8-bit source plane -> 9 / 10-bit plane (swscale_unscaled.c:946-971): limited-range luma and both chroma
// planes are plain shifts; -> 16-bit plane (:984-992): the byte twice
__global__ void __launch_bounds__(256)
sws_copy_plane_up_kernel(const uint8_t *__restrict__ src, int srcStride, size_t srcFrame, uint8_t *__restrict__ dst, int dstStride, size_t dstFrame,
                         int w, int h, int shift, int be)
{
    const int x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y;
    if (x >= w) return;
    const int v = src[blockIdx.z * srcFrame + (size_t)y * srcStride + x];
    reinterpret_cast<uint16_t *>(dst + blockIdx.z * dstFrame + (size_t)y * dstStride)[x] = (uint16_t)swap16_if(shift == 8 ? v * 257 : v << shift, be);
}

// yuyvToYuv422Wrapper / uyvyToYuv422Wrapper -> yuyvtoyuv422_c / uyvytoyuv422_c (rgb2rgb_template.c:873-888,912-927): one thread per pixel pair
__global__ void __launch_bounds__(256)
sws_yuyv_yuv422p_kernel(const uint8_t *__restrict__ src, int srcStride, size_t srcFrame, uint8_t *__restrict__ Y, uint8_t *__restrict__ U,
                        uint8_t *__restrict__ V, int yStride, int cStride, size_t yFrame, size_t uFrame, size_t vFrame, int w, int h, int uyvy)
{
    const int i = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y;
    if (2 * i >= w) return;
    const size_t f = blockIdx.z;
    const uint8_t *s = src + f * srcFrame + (size_t)y * srcStride + 4 * i;
    uint8_t *dy = Y + f * yFrame + (size_t)y * yStride + 2 * i;
    const int yo = uyvy ? 1 : 0, co = uyvy ? 0 : 1;
    const bool second = 2 * i + 1 < w;
    dy[0] = s[yo];
    if (second) dy[1] = s[2 + yo];
    U[f * uFrame + (size_t)y * cStride + i] = s[co];
    V[f * vFrame + (size_t)y * cStride + i] = (second || 4 * i + 4 <= srcStride || y < h - 1) ? s[2 + co] : s[co];
}

// ---------------------------------------------------------------------------------------------------
// pixel formats
// ---------------------------------------------------------------------------------------------------
// AV_PIX_FMT_* values, libavutil/pixfmt.h (the only place the scaler spells them out)
enum {
    PIX_YUV420P = 0, PIX_YUYV422 = 1, PIX_RGB24 = 2, PIX_BGR24 = 3, PIX_YUV422P = 4, PIX_YUV444P = 5, PIX_YUV410P = 6, PIX_YUV411P = 7,
    PIX_GRAY8 = 8, PIX_PAL8 = 11, PIX_YUVJ420P = 12, PIX_YUVJ422P = 13, PIX_YUVJ444P = 14, PIX_UYVY422 = 15, PIX_NV12 = 23, PIX_NV21 = 24,
    PIX_ARGB = 25, PIX_RGBA = 26, PIX_ABGR = 27, PIX_BGRA = 28, PIX_YUV440P = 31, PIX_YUVJ440P = 32, PIX_YUVA420P = 33,
    PIX_RGB48BE = 34, PIX_RGB48LE = 35, PIX_RGB565BE = 36, PIX_RGB565LE = 37, PIX_RGB555BE = 38, PIX_RGB555LE = 39,
    PIX_BGR565BE = 40, PIX_BGR565LE = 41, PIX_BGR555BE = 42, PIX_BGR555LE = 43, PIX_YUV420P16LE = 47, PIX_YUV420P16BE = 48,
    PIX_YUV422P16LE = 49, PIX_YUV422P16BE = 50, PIX_YUV444P16LE = 51, PIX_YUV444P16BE = 52, PIX_RGB444LE = 54, PIX_RGB444BE = 55,
    PIX_BGR444LE = 56, PIX_BGR444BE = 57, PIX_BGR48BE = 59, PIX_BGR48LE = 60, PIX_YUV420P9BE = 61, PIX_YUV420P9LE = 62,
    PIX_YUV420P10BE = 63, PIX_YUV420P10LE = 64, PIX_YUV422P10BE = 65, PIX_YUV422P10LE = 66, PIX_YUV444P9BE = 67, PIX_YUV444P9LE = 68,
    PIX_YUV444P10BE = 69, PIX_YUV444P10LE = 70, PIX_YUV422P9BE = 71, PIX_YUV422P9LE = 72,
};
enum PixFam { FAM_YUV, FAM_NV, FAM_PK422, FAM_RGB24, FAM_RGB32, FAM_RGB16, FAM_RGB48, FAM_GRAY, FAM_PAL8 };
enum { IN = 1, OUT = 2 };     // the sides a format is taken over on

struct PixFmt {
    int fmt, side; PixFam fam;
    int hs, vs;               // chroma sub-sampling, log2 (libavutil/pixdesc.c log2_chroma_w / _h; rgb sources: chosen per context)
    int bits, be, full;       // sample depth; 16-bit planar samples stored big-endian; full range (yuvj, handle_jpeg, utils.c:855-873)
    int bpp;                  // bytes per pixel of a packed format
    int r, g, b, a;           // byte of each channel in a 24 / 32-bit rgb pixel (-1: none)
    int pk422, rgb16, rgb48, chrStep, slot;     // the SwsDev codes; SwsSlotView::target (-1 planar)
    int fold;                 // the format the conversion runs as: yuvj -> yuv, yuva420p -> yuv420p (its alpha plane is never read,
                              // swscale_unscaled.c:1041-1153), 9 / 10 / 16-bit -> its 8-bit layout, gray8 source -> the luma of a 4:4:4 picture
};
#define YUV(f, s, hs, vs, bits, be, full, fold) { f, s, FAM_YUV, hs, vs, bits, be, full, 0, -1, -1, -1, -1, 0, 0, 0, 1, -1, fold }
#define RGB(f, fam, bpp, r, g, b, a, rgb16, rgb48, slot) { f, fam == FAM_RGB16 || fam == FAM_RGB48 ? OUT : IN | OUT, fam, 1, 0, 8, 0, 0, bpp, r, g, b, a, 0, rgb16, rgb48, 1, slot, f }
static const PixFmt PIXFMTS[] = {
    YUV(PIX_YUV420P, IN | OUT, 1, 1, 8, 0, 0, PIX_YUV420P),        YUV(PIX_YUVJ420P, IN | OUT, 1, 1, 8, 0, 1, PIX_YUV420P),
    YUV(PIX_YUV422P, IN | OUT, 1, 0, 8, 0, 0, PIX_YUV422P),        YUV(PIX_YUVJ422P, IN | OUT, 1, 0, 8, 0, 1, PIX_YUV422P),
    YUV(PIX_YUV444P, IN | OUT, 0, 0, 8, 0, 0, PIX_YUV444P),        YUV(PIX_YUVJ444P, IN | OUT, 0, 0, 8, 0, 1, PIX_YUV444P),
    YUV(PIX_YUV440P, IN | OUT, 0, 1, 8, 0, 0, PIX_YUV440P),        YUV(PIX_YUVJ440P, IN | OUT, 0, 1, 8, 0, 1, PIX_YUV440P),
    YUV(PIX_YUV410P, IN | OUT, 2, 2, 8, 0, 0, PIX_YUV410P),        YUV(PIX_YUV411P, IN | OUT, 2, 0, 8, 0, 0, PIX_YUV411P),
    YUV(PIX_YUVA420P, IN, 1, 1, 8, 0, 0, PIX_YUV420P),
    YUV(PIX_YUV420P9LE, IN | OUT, 1, 1, 9, 0, 0, PIX_YUV420P),     YUV(PIX_YUV420P9BE, IN | OUT, 1, 1, 9, 1, 0, PIX_YUV420P),
    YUV(PIX_YUV420P10LE, IN | OUT, 1, 1, 10, 0, 0, PIX_YUV420P),   YUV(PIX_YUV420P10BE, IN | OUT, 1, 1, 10, 1, 0, PIX_YUV420P),
    YUV(PIX_YUV420P16LE, IN | OUT, 1, 1, 16, 0, 0, PIX_YUV420P),   YUV(PIX_YUV420P16BE, IN | OUT, 1, 1, 16, 1, 0, PIX_YUV420P),
    YUV(PIX_YUV422P9LE, IN | OUT, 1, 0, 9, 0, 0, PIX_YUV422P),     YUV(PIX_YUV422P9BE, IN | OUT, 1, 0, 9, 1, 0, PIX_YUV422P),
    YUV(PIX_YUV422P10LE, IN | OUT, 1, 0, 10, 0, 0, PIX_YUV422P),   YUV(PIX_YUV422P10BE, IN | OUT, 1, 0, 10, 1, 0, PIX_YUV422P),
    YUV(PIX_YUV422P16LE, IN | OUT, 1, 0, 16, 0, 0, PIX_YUV422P),   YUV(PIX_YUV422P16BE, IN | OUT, 1, 0, 16, 1, 0, PIX_YUV422P),
    YUV(PIX_YUV444P9LE, IN | OUT, 0, 0, 9, 0, 0, PIX_YUV444P),     YUV(PIX_YUV444P9BE, IN | OUT, 0, 0, 9, 1, 0, PIX_YUV444P),
    YUV(PIX_YUV444P10LE, IN | OUT, 0, 0, 10, 0, 0, PIX_YUV444P),   YUV(PIX_YUV444P10BE, IN | OUT, 0, 0, 10, 1, 0, PIX_YUV444P),
    YUV(PIX_YUV444P16LE, IN | OUT, 0, 0, 16, 0, 0, PIX_YUV444P),   YUV(PIX_YUV444P16BE, IN | OUT, 0, 0, 16, 1, 0, PIX_YUV444P),
    // semi-planar: the luma plane and one plane of interleaved chroma (chrStep 2 in the kernels)
    { PIX_NV12, IN | OUT, FAM_NV, 1, 1, 8, 0, 0, 0, -1, -1, -1, -1, 0, 0, 0, 2, -1, PIX_NV12 },
    { PIX_NV21, IN | OUT, FAM_NV, 1, 1, 8, 0, 0, 0, -1, -1, -1, -1, 0, 0, 0, 2, -1, PIX_NV21 },
    { PIX_YUYV422, IN | OUT, FAM_PK422, 1, 0, 8, 0, 0, 2, -1, -1, -1, -1, 1, 0, 0, 1, 2, PIX_YUYV422 },
    { PIX_UYVY422, IN | OUT, FAM_PK422, 1, 0, 8, 0, 0, 2, -1, -1, -1, -1, 2, 0, 0, 1, 3, PIX_UYVY422 },
    // gray8: one component (pixdesc); as a destination it becomes a planar stand-in chosen per context
    { PIX_GRAY8, IN | OUT, FAM_GRAY, 0, 0, 8, 0, 0, 1, -1, -1, -1, -1, 0, 0, 0, 1, -1, PIX_YUV444P },
    { PIX_PAL8, IN, FAM_PAL8, 0, 0, 8, 0, 0, 1, -1, -1, -1, -1, 0, 0, 0, 1, -1, PIX_PAL8 },
    RGB(PIX_RGB24, FAM_RGB24, 3, 0, 1, 2, -1, 0, 0, 0),  RGB(PIX_BGR24, FAM_RGB24, 3, 2, 1, 0, -1, 0, 0, 1),
    RGB(PIX_ARGB, FAM_RGB32, 4, 1, 2, 3, 0, 0, 0, 4),    RGB(PIX_RGBA, FAM_RGB32, 4, 0, 1, 2, 3, 0, 0, 5),
    RGB(PIX_ABGR, FAM_RGB32, 4, 3, 2, 1, 0, 0, 0, 6),    RGB(PIX_BGRA, FAM_RGB32, 4, 2, 1, 0, 3, 0, 0, 7),
    // 15 / 16 / 12 bpp: SwsDev::rgb16 1 rgb565 2 bgr565 3 rgb555 4 bgr555 5 rgb444 6 bgr444, + 8 big-endian; 48 bpp: SwsDev::rgb48 1 rgb 2 bgr, + 8 big-endian
    RGB(PIX_RGB565LE, FAM_RGB16, 2, -1, -1, -1, -1, 1, 0, -1),  RGB(PIX_RGB565BE, FAM_RGB16, 2, -1, -1, -1, -1, 1 | 8, 0, -1),
    RGB(PIX_BGR565LE, FAM_RGB16, 2, -1, -1, -1, -1, 2, 0, -1),  RGB(PIX_BGR565BE, FAM_RGB16, 2, -1, -1, -1, -1, 2 | 8, 0, -1),
    RGB(PIX_RGB555LE, FAM_RGB16, 2, -1, -1, -1, -1, 3, 0, -1),  RGB(PIX_RGB555BE, FAM_RGB16, 2, -1, -1, -1, -1, 3 | 8, 0, -1),
    RGB(PIX_BGR555LE, FAM_RGB16, 2, -1, -1, -1, -1, 4, 0, -1),  RGB(PIX_BGR555BE, FAM_RGB16, 2, -1, -1, -1, -1, 4 | 8, 0, -1),
    RGB(PIX_RGB444LE, FAM_RGB16, 2, -1, -1, -1, -1, 5, 0, -1),  RGB(PIX_RGB444BE, FAM_RGB16, 2, -1, -1, -1, -1, 5 | 8, 0, -1),
    RGB(PIX_BGR444LE, FAM_RGB16, 2, -1, -1, -1, -1, 6, 0, -1),  RGB(PIX_BGR444BE, FAM_RGB16, 2, -1, -1, -1, -1, 6 | 8, 0, -1),
    RGB(PIX_RGB48LE, FAM_RGB48, 6, -1, -1, -1, -1, 0, 1, -1),   RGB(PIX_RGB48BE, FAM_RGB48, 6, -1, -1, -1, -1, 0, 1 | 8, -1),
    RGB(PIX_BGR48LE, FAM_RGB48, 6, -1, -1, -1, -1, 0, 2, -1),   RGB(PIX_BGR48BE, FAM_RGB48, 6, -1, -1, -1, -1, 0, 2 | 8, -1),
};
#undef YUV
#undef RGB

// the row of a format taken over on `side`, null for anything else
static const PixFmt *pixfmt(int fmt, int side)
{
    for (const PixFmt &f : PIXFMTS) if (f.fmt == fmt) return (f.side & side) ? &f : nullptr;
    return nullptr;
}
static bool is_planar(const PixFmt *f) { return f->fam == FAM_YUV || f->fam == FAM_NV; }
static bool is_packed_src(const PixFmt *f) { return f->fam == FAM_PK422 || f->fam == FAM_RGB24 || f->fam == FAM_RGB32 || f->fam == FAM_PAL8; }

// ---------------------------------------------------------------------------------------------------
// context
// ---------------------------------------------------------------------------------------------------
// The conversion a context runs, chosen once by choose_route() like the reference picks its SwsFunc (utils.c:1043-1054,
// swscale_unscaled.c:1040-1176).  A packed or semi-planar source reaches the planar routes through a pre-pass (the input readers,
// input.c, or the nv split), and a 32-bit rgb destination through an expansion of their rgb24 output (run_frames).
enum Route {
    R_SCALE,            // swscale(): the tile kernel or the two passes
    R_FUSED,            // same-size yuv420p -> 24 / 32-bit rgb with identity filters and a 4-tap vertical chroma filter: one kernel
    R_RGB48,            // 48-bit rgb: sws_rgb48_kernel straight from the source planes
    R_TABLE,            // the unscaled yuv2rgb table converter (yuv2rgb.c), same-size rgb without SWS_ACCURATE_RND and an even height
    R_COPY,             // planarCopyWrapper, nv12ToPlanarWrapper
    R_RGB_COPY,         // rgb24 / bgr24 to itself
    R_RGB24_SWAP,       // rgb24 <-> bgr24
    R_BGR24_YV12,       // rgb24toyv12_c
    R_YUYV_420P,        // yuyv422 / uyvy422 -> yuv420p
    R_YUYV_422P,        // yuyv422 / uyvy422 -> yuv422p
    R_RGB_REMAP,        // rgbToRgbWrapper's byte converters: 24 / 32-bit rgb pairs with 32 bits on at least one side
    R_GRAY_RGB,         // palToRgbWrapper with gray8's pseudo-palette r = g = b = sample
    R_PAL8_RGB,         // palToRgbWrapper
    R_422_FROM_422P,    // yuv422p -> yuyv422 / uyvy422
    R_422_FROM_420P,    // yuv420p -> yuyv422 / uyvy422 (fast-bilinear / point flags only)
    R_422_COPY,         // yuyv422 / uyvy422 to itself
    R_NV_INTERLEAVE,    // planarToNv12Wrapper
};
static const struct RouteFacts {
    int plan;           // sws_debug_plan_cuda out[0]
    bool planar;        // runs on yuv planes: pre-pass for packed / semi-planar sources, expansion for 32-bit rgb destinations
    bool rowMapped;     // output row y comes from source row y: a slice completes its own rows
    int chrAlign;       // log2 of the source rows a slice must start on, at least (it also works on whole row pairs)
    bool tables;        // reads the yuv -> rgb colour tables
} ROUTES[] = {
    { 4, true, false, 0, true },  { 3, true, false, 0, true },  { 4, true, false, 0, true },  { 2, true, true, 1, true },
    { 1, false, true, 0, true },  { 5, false, true, 0, false }, { 5, false, true, 0, false }, { 5, false, true, 1, false },
    { 5, false, true, 0, false }, { 5, false, true, 0, false }, { 5, false, true, 0, false }, { 5, false, true, 0, false },
    { 5, false, true, 0, false }, { 6, false, true, 0, true },  { 6, false, true, 1, true },  { 6, false, true, 0, true },
    { 7, false, true, 0, true },
};

struct SwsCudaContext {
    SwsGeometry g;
    FilterBank hLum, hChr, vLum, vChr;
    RgbConstants k;
    const PixFmt *srcFmt, *dstFmt;   // the formats the caller named
    const PixFmt *S, *D;             // the formats the conversion runs as (PixFmt::fold; a gray8 destination: the planar stand-in, a
                                     // destination keeps its own depth)
    Route route;
    bool fast_ok = false;       // the fused interior kernel's host-side preconditions on the filter bank hold
    void *d_tables = nullptr;   // all filter banks in one device allocation
    void *d_pair_taps = nullptr; // SwsPairTaps[dstH / 2] for the dp4a fused kernel (fast_ok only)
    void *d_pair_taps_t = nullptr; // SwsPairTapsT[dstH / 2] for the TMA fused kernel (tma_ok only)
    bool tma_ok = false;        // every four-pair tile of the TMA kernel reaches at most eight chroma lines
    // the TMA kernel's tile counters (tma_ok only): one for launches on the caller's stream, one for each of `streams`.  Launches that
    // share a counter must be ordered, so the device-pointer calls of a context go to one stream, or to streams the caller orders.
    int *d_tickets = nullptr;
    SwsDev dev;
    int16_t *d_lum = nullptr, *d_chrU = nullptr, *d_chrV = nullptr;   // general path line planes
    int lumStridePx = 0, chrStridePx = 0;
    uint8_t *d_pal = nullptr;   // pal8 sources through the host-pointer call: the caller's palette (256 x 4 bytes)
    uint8_t *d_rgb = nullptr; size_t rgb_bytes = 0;     // the rgb24 picture a 32-bit destination is expanded from
    int srcRange = 0;           // 1 = full-range (JPEG) source, sws_setColorspaceDetails / a yuvj source format
    int rangeConv = 0;          // yuv destination of the other range: 1 lum / chrRangeFromJpeg_c, 2 lum / chrRangeToJpeg_c on the hscaled lines (two-pass path)
    // gray8 destination: the luma plane of the planar conversion (swscale.c:618-630 skips the chroma of a gray destination, the unscaled
    // copy takes plane 0 only, swscale_unscaled.c:1155); the chroma planes go to scratch nobody reads
    uint8_t *d_gray[2] = { nullptr, nullptr }; int grayPitch = 0;
    std::vector<uint8_t> h_gray[2];
    uint8_t *d_nv = nullptr; size_t nv_bytes = 0;   // the planes the pre-pass of a batch writes (split nv chroma, reader output)
    int2 *d_tile_win = nullptr; size_t tileChrWinOff = 0;
    int tileLumRows = 0, tileChrRows = 0;  // fused-tile general path: shared-memory line capacity; 0 = window too large, two passes
    // staging for the host-pointer sws_scale_cuda()
    uint8_t *d_src = nullptr, *d_dst = nullptr; size_t src_bytes = 0, dst_bytes = 0;
    cudaStream_t streams[3] = {}; bool streams_ok = false;
    // slices (sws_scale_cuda_sliced): the source rows received so far, the next expected source row, the output rows already returned
    std::vector<uint8_t> sliceSrc[3]; int slicePitch[3] = { 0, 0, 0 }; int sliceNextY = 0, sliceDstY = 0;
};

static void destroy(SwsCudaContext *c)
{
    if (!c) return;
    if (c->streams_ok) for (int i = 0; i < 3; i++) cudaStreamDestroy(c->streams[i]);
    cudaFree(c->d_pal); cudaFree(c->d_tables); cudaFree(c->d_pair_taps); cudaFree(c->d_pair_taps_t); cudaFree(c->d_tickets); cudaFree(c->d_nv); cudaFree(c->d_rgb); cudaFree(c->d_tile_win); cudaFree(c->d_lum); cudaFree(c->d_chrU); cudaFree(c->d_chrV); cudaFree(c->d_src); cudaFree(c->d_dst); cudaFree(c->d_gray[0]); cudaFree(c->d_gray[1]);
    delete c;
}

static bool is_identity(const FilterBank &b, int one)
{
    if (b.size != 1) return false;
    for (int i = 0; i < b.n; i++) if (b.coef[i] != one || b.pos[i] != i) return false;
    return true;
}

// a device copy of a host table; the sticky error is set on failure
static int upload(void **d, const void *h, size_t bytes)
{
    if (cudaMalloc(d, bytes) != cudaSuccess || cudaMemcpy(*d, h, bytes, cudaMemcpyHostToDevice) != cudaSuccess) {
        set_error("sws_getContext_cuda", cudaGetLastError()); return -1;
    }
    return 0;
}

// a scratch buffer of at least `need` bytes; an earlier batch on `st` may still use the old one
static int grow(uint8_t *&buf, size_t &bytes, size_t need, cudaStream_t st, const char *where)
{
    if (bytes >= need) return 0;
    AVB_CUDA(cudaStreamSynchronize(st), where);
    cudaFree(buf); buf = nullptr; bytes = 0;
    AVB_CUDA(cudaMalloc(&buf, need), where);
    bytes = need;
    return 0;
}

static int upload_tables(SwsCudaContext *c)
{
    const FilterBank *banks[4] = { &c->hLum, &c->hChr, &c->vLum, &c->vChr };
    size_t off[8], total = 0;
    for (int b = 0; b < 4; b++) {
        off[2 * b] = total;     total += (banks[b]->coef.size() * 2 + 255) & ~(size_t)255;
        off[2 * b + 1] = total; total += (banks[b]->pos.size() * 4 + 255) & ~(size_t)255;
    }
    AVB_CUDA(cudaMalloc(&c->d_tables, total), "sws:tables");
    uint8_t *base = (uint8_t *)c->d_tables;
    for (int b = 0; b < 4; b++) {
        AVB_CUDA(cudaMemcpy(base + off[2 * b], banks[b]->coef.data(), banks[b]->coef.size() * 2, cudaMemcpyHostToDevice), "sws:tables");
        AVB_CUDA(cudaMemcpy(base + off[2 * b + 1], banks[b]->pos.data(), banks[b]->pos.size() * 4, cudaMemcpyHostToDevice), "sws:tables");
    }
    SwsDev &d = c->dev;
    const PixFmt *D = c->D;
    d.srcW = c->g.srcW; d.srcH = c->g.srcH; d.dstW = c->g.dstW; d.dstH = c->g.dstH;
    d.chrSrcW = c->g.chrSrcW; d.chrSrcH = c->g.chrSrcH; d.chrDstW = c->g.chrDstW; d.chrDstH = c->g.chrDstH;
    d.hLumSize = c->hLum.size; d.hChrSize = c->hChr.size; d.vLumSize = c->vLum.size; d.vChrSize = c->vChr.size;
    d.hLumF = (const int16_t *)(base + off[0]); d.hLumP = (const int32_t *)(base + off[1]);
    d.hChrF = (const int16_t *)(base + off[2]); d.hChrP = (const int32_t *)(base + off[3]);
    d.vLumF = (const int16_t *)(base + off[4]); d.vLumP = (const int32_t *)(base + off[5]);
    d.vChrF = (const int16_t *)(base + off[6]); d.vChrP = (const int32_t *)(base + off[7]);
    d.k = c->k;
    d.bgr = D->fmt == PIX_BGR24 || (D->rgb48 & 7) == 2;
    d.full = (c->g.flags & SWS_FULL_CHR_H_INT) != 0 && !is_planar(D);
    d.dstBits = D->bits; d.dstBE = D->be; d.chrStep = D->chrStep; d.pk422 = D->pk422; d.rgb16 = D->rgb16; d.rgb48 = D->rgb48; d.srcGray = c->srcFmt->fam == FAM_GRAY;
    d.srcBits = c->srcFmt->bits; d.srcBE = c->srcFmt->be; d.dither = c->srcFmt->bits > 8;
    return 0;
}

// The route of a context that passed every refusal, its filter banks designed
static Route choose_route(const SwsCudaContext *c, int flags, bool unscaled, bool usesFilter, bool grayPal, bool rgb2rgb)
{
    const PixFmt *S = c->S, *D = c->D;
    const bool rgb = !is_planar(D), bits8 = c->srcFmt->bits == 8, srcGray = c->srcFmt->fam == FAM_GRAY;
    if (D->pk422 && unscaled && !usesFilter && !c->rangeConv && bits8) {              // swscale_unscaled.c:1123-1139,1152-1176
        if (S->fmt == PIX_YUV422P) return R_422_FROM_422P;
        if (S->fmt == PIX_YUV420P && (flags & (SWS_FAST_BILINEAR | SWS_POINT))) return R_422_FROM_420P;
        if (S->fmt == D->fmt) return R_422_COPY;
    }
    if (D->fam == FAM_NV && S->fmt == PIX_YUV420P && unscaled && !c->rangeConv && bits8) return R_NV_INTERLEAVE;     // swscale_unscaled.c:1040-1044
    if (unscaled && !usesFilter) {                            // swscale_unscaled.c:1063-1072,1140-1145,1152-1176 (yuv destinations: only with equal ranges, utils.c:1043-1044)
        if (S->fam == FAM_PAL8 && (D->fam == FAM_RGB24 || D->fam == FAM_RGB32)) return R_PAL8_RGB;       // swscale_unscaled.c:1114-1121
        if (grayPal) return R_GRAY_RGB;
        if (rgb2rgb) return R_RGB_REMAP;
        if (S->fam == FAM_RGB24 && rgb && !D->pk422) return S->fmt == D->fmt ? R_RGB_COPY : R_RGB24_SWAP;
        // (a gray8 destination is served through a planar stand-in: the reference installs these converters for real yuv420p / yuv422p destinations only)
        if (!c->rangeConv && c->dstFmt->fam != FAM_GRAY) {
            if (S->fmt == PIX_BGR24 && D->fmt == PIX_YUV420P && !(flags & SWS_ACCURATE_RND)) return R_BGR24_YV12;
            if (S->fam == FAM_PK422 && D->fmt == PIX_YUV420P) return R_YUYV_420P;
            if (S->fam == FAM_PK422 && D->fmt == PIX_YUV422P) return R_YUYV_422P;
        }
    }
    // planarCopyWrapper for planar -> planar of the same size and sub-sampling (swscale_unscaled.c:1152-1176), nv12ToPlanarWrapper for
    // nv12 / nv21 -> yuv420p (:1046-1049); other nv12 destinations go through swscale()
    if (D->fam == FAM_YUV && (S->fam == FAM_YUV || (S->fam == FAM_NV && D->fmt == PIX_YUV420P)) && unscaled && ((S->hs == D->hs && S->vs == D->vs) || srcGray) &&
        !c->rangeConv && !usesFilter && bits8) return R_COPY;
    // swscale_unscaled.c:1051-1055; the table converter only exists for planar sources (an nv12 frame goes through swscale())
    if ((S->fmt == PIX_YUV420P || S->fmt == PIX_YUV422P) && rgb && !D->pk422 && unscaled && !(flags & SWS_ACCURATE_RND) && !(c->g.dstH & 1) && !usesFilter && bits8) return R_TABLE;
    if (D->rgb48) return R_RGB48;
    if (bits8 && !srcGray && rgb && !D->pk422 && !D->rgb16 && !(flags & SWS_FULL_CHR_H_INT) && !(c->g.flags & SWS_FAST_BILINEAR) && is_identity(c->hLum, 1 << 14) &&
        is_identity(c->hChr, 1 << 14) && is_identity(c->vLum, 1 << 12) && c->vChr.size == 4) return R_FUSED;
    return R_SCALE;
}

struct SwsFilterView { const SwsVec *lumH, *lumV, *chrH, *chrV; };      // libswscale/swscale.h:112-117 (a SwsVector is { double *coeff; int length; })
static SwsCudaContext *make_context(int srcW, int srcH, int srcFormat, int dstW, int dstH, int dstFormat, int flags,
                                    const double *param, bool device_side, const void *srcFilter = nullptr, const void *dstFilter = nullptr)
{
    static const SwsFilterView noFilter = { nullptr, nullptr, nullptr, nullptr };
    const SwsFilterView &sf = srcFilter ? *(const SwsFilterView *)srcFilter : noFilter, &df = dstFilter ? *(const SwsFilterView *)dstFilter : noFilter;
    auto longer = [](const SwsVec *v) { return v && v->length > 1; };
    // usesVFilter / usesHFilter (utils.c:974-981): with either, no unscaled special converter is installed (:1043)
    const bool usesFilter = longer(sf.lumV) || longer(sf.chrV) || longer(df.lumV) || longer(df.chrV) || longer(sf.lumH) || longer(sf.chrH) || longer(df.lumH) || longer(df.chrH);
    const bool unscaled = srcW == dstW && srcH == dstH;
    const char *err = nullptr;
    const PixFmt *srcIn = pixfmt(srcFormat, IN), *dstIn = pixfmt(dstFormat, OUT);
    const PixFmt *S = srcIn ? pixfmt(srcIn->fold, IN) : nullptr, *D = dstIn && dstIn->full ? pixfmt(dstIn->fold, OUT) : dstIn;
    const int srcRange = srcIn ? srcIn->full : 0, dstRange = dstIn ? dstIn->full : 0, srcBits = srcIn ? srcIn->bits : 8;
    const bool srcGray = srcIn && srcIn->fam == FAM_GRAY, gray = dstIn && dstIn->fam == FAM_GRAY;
    // yuva420p: the alpha plane is read only when the destination has alpha too (utils.c:1244, yuv2rgb.c:870)
    if (srcIn && srcIn->fmt == PIX_YUVA420P && D && D->fam == FAM_RGB32) {
        set_error_msg("sws_getContext_cuda", "yuva420p to a destination with alpha (the alpha plane is scaled too) is not taken over"); return nullptr;
    }
    bool grayPal = false;
    if (srcGray) {
        const char *why = nullptr;
        if (dstRange) why = "gray8 to a full-range yuvj destination (range conversion) is not taken over";
        else if (D && D->fam == FAM_NV) why = "gray8 to nv12 / nv21 is not taken over (the reference's plane copy fills half of the interleaved chroma row)";
        if (why) { set_error_msg("sws_getContext_cuda", why); return nullptr; }
        // same size to 24 / 32-bit rgb: palToRgbWrapper with the pseudo-palette r = g = b = sample (swscale_unscaled.c:342-384,1114-1121,1257-1259)
        grayPal = unscaled && D && (D->fam == FAM_RGB24 || D->fam == FAM_RGB32);
    }
    // gray8 destination: the luma plane of the conversion to a planar yuv picture -- of the source's own sub-sampling when the source is
    // planar 8-bit yuv, so that the same-size case is the reference's plane copy for every such source (isPlanarYUV(src) && isGray(dst),
    // swscale_unscaled.c:1155) -- whose chroma planes are written to scratch
    if (gray) D = pixfmt(S && S->fam == FAM_YUV ? S->fmt : PIX_YUV420P, OUT);
    if (!D) {
        set_error_msg("sws_getContext_cuda", "destinations taken over: gray8, rgb24, bgr24, argb, rgba, abgr, bgra, rgb48 / bgr48 (LE and BE), rgb565 / bgr565 / rgb555 / bgr555 / rgb444 / bgr444 (LE and BE), yuyv422, uyvy422, nv12, nv21, planar yuv 420p 422p 444p 410p 411p 440p, 9 / 10 / 16-bit 420p 422p 444p (LE and BE)");
        return nullptr;
    }
    const bool planar = is_planar(D), rgb = !planar;
    if (D->pk422 || D->rgb16 || D->rgb48) flags &= ~SWS_FULL_CHR_H_INT;        // only 24 / 32-bit packed RGB knows the flag (utils.c:998-1014)
    if (flags & 0x30000) {                                    // SWS_SRC_V_CHR_DROP_MASK (utils.c:1016-1019, swscale.c:383-384)
        set_error_msg("sws_getContext_cuda", "SWS_SRC_V_CHR_DROP (skipping source chroma lines) is not taken over"); return nullptr;
    }
    if (!S) {
        set_error_msg("sws_getContext_cuda", "sources taken over: planar 8-bit yuv (420p 422p 444p 410p 411p 440p, yuvj, yuva420p), gray8, 9 / 10 / 16-bit planar yuv, nv12, nv21, yuyv422, uyvy422, rgb24, bgr24, argb, rgba, abgr, bgra");
        return nullptr;
    }
    const bool srcRgb = S->fam == FAM_RGB24, src32 = S->fam == FAM_RGB32, srcYuy = S->fam == FAM_PK422, srcPal = S->fam == FAM_PAL8, srcNV = S->fam == FAM_NV;
    const bool dst32 = D->fam == FAM_RGB32, dstNV = D->fam == FAM_NV;
    int hs = S->hs, vs = S->vs;
    if (srcRgb || src32) {      // utils.c:1021-1034: every other pixel for chroma unless told / forced otherwise
        const int chrDstHSub = planar ? D->hs : (flags & SWS_FULL_CHR_H_INT) ? 0 : 1;
        hs = (!(flags & SWS_FULL_CHR_H_INP) && ((dstW >> chrDstHSub) <= (srcW >> 1) || (flags & SWS_FAST_BILINEAR))) ? 1 : 0;
    }
    if (srcNV && dstNV && unscaled) {
        set_error_msg("sws_getContext_cuda", "nv12 / nv21 -> nv12 / nv21 of the same size (the reference's plane copy skips the chroma plane there) is not taken over"); return nullptr;
    }
    // same size, packed rgb on both sides, 32 bits on at least one: rgbToRgbWrapper's byte converters (swscale_unscaled.c:590-705), a channel remap
    const bool rgb2rgb = unscaled && !usesFilter && (srcRgb || src32) && (D->fam == FAM_RGB24 || dst32) && (src32 || dst32);
    if (src32 && !rgb2rgb && (dst32 || (unscaled && !planar && !D->pk422))) {
        // 32 -> 32 bit at another size: the reference scales the alpha plane too; same size -> 16 / 48-bit rgb: other converter families
        set_error_msg("sws_getContext_cuda", "32-bit rgb source: planar yuv destinations, scaled rgb24 / bgr24 and same-size 24 / 32-bit rgb are taken over"); return nullptr;
    }
    if (D->fmt == PIX_ABGR && (flags & SWS_FULL_CHR_H_INT) && !grayPal && !rgb2rgb && !(srcPal && unscaled && !usesFilter)) {      // (the unscaled converters never reach that output function)  // output.c:1231-1237 advances the pointer twice per abgr pixel and runs off the row
        set_error_msg("sws_getContext_cuda", "abgr with SWS_FULL_CHR_H_INT: the reference's output function overruns the destination; there is no result to match");
        return nullptr;
    }
    if (srcRgb && unscaled && (D->fmt == PIX_ARGB || D->fmt == PIX_ABGR)) {
        // rgbToRgbWrapper moves the 4-byte writer one byte into the row for these two (ALT32_CORR, swscale_unscaled.c:691-692): the first alpha byte is
        // never written and the last write lands past the row
        set_error_msg("sws_getContext_cuda", "rgb24 / bgr24 -> argb / abgr of the same size: the reference's converter writes past the row; there is no result to match");
        return nullptr;
    }
    if (S->fmt == PIX_BGR24 && D->fmt == PIX_YUV420P && !gray && unscaled && !(flags & SWS_ACCURATE_RND) && (srcH & 1) && srcRange == dstRange) {
        set_error_msg("sws_getContext_cuda", "bgr24 -> yuv420p of the same size without SWS_ACCURATE_RND is the reference's rgb24toyv12, which needs an even height");
        return nullptr;
    }
    if (S->fmt == PIX_YUV410P && D->fmt == PIX_YUV420P && unscaled && !(flags & SWS_BITEXACT) && srcRange == dstRange) {
        set_error_msg("sws_getContext_cuda", "yuv410p -> yuv420p of the same size without SWS_BITEXACT is the reference's yvu9ToYv12Wrapper: not taken over");
        return nullptr;
    }
    if (D->rgb16) {
        // the 15 / 16 / 12-bpp destinations exist where swscale()'s packed output stage runs (yuv2rgb16_X / _2 / _1 ..., output.c:1321-1326);
        // the reference's other routes to them are separate converter families that are not taken over
        const char *why = nullptr;
        if (srcRgb || src32 || srcYuy || srcPal) why = "15 / 16 / 12-bpp rgb destinations are taken over for planar / semi-planar yuv sources only";
        else if ((S->fmt == PIX_YUV420P || S->fmt == PIX_YUV422P) && unscaled && !(flags & SWS_ACCURATE_RND) && !(dstH & 1) && !usesFilter && srcBits == 8)
            why = "same-size yuv -> 15 / 16 / 12-bpp rgb without SWS_ACCURATE_RND is the reference's ordered-dither table converter (yuv2rgb.c:377-573): not taken over";
        else if (usesFilter) why = "SwsFilter vectors with a 15 / 16 / 12-bpp destination are not taken over";
        if (why) { set_error_msg("sws_getContext_cuda", why); return nullptr; }
    }
    if (srcGray) {
        const char *why = nullptr;
        if (usesFilter) why = "SwsFilter vectors with a gray8 source are not taken over";
        else if (planar && D->bits == 16) why = "gray8 to a 16-bit planar destination is not taken over";
        else if (planar && D->bits != 8 && unscaled) why = "gray8 to a 9 / 10-bit planar destination of the same size (planarCopyWrapper's fill_plane9or10) is not taken over";
        if (why) { set_error_msg("sws_getContext_cuda", why); return nullptr; }
    }
    if (D->rgb48) {
        // 48-bit destinations: the packed output stage on hScale8To19_c lines, and the unscaled table converter; planar 8-bit yuv sources
        const char *why = nullptr;
        if (srcRgb || src32 || srcYuy || srcPal || srcNV) why = "48-bit rgb destinations are taken over for planar 8-bit yuv sources only";
        else if (srcBits > 8) why = "9 / 10 / 16-bit source to a 48-bit rgb destination (hScale16To19_c lines) is not taken over";
        else if (usesFilter) why = "SwsFilter vectors with a 48-bit rgb destination are not taken over";
        if (why) { set_error_msg("sws_getContext_cuda", why); return nullptr; }
    }
    {   // a shifted / asymmetric vertical vector makes the reference's last output rows depend on stale lines of its ring buffer (measured:
        // port and product, which clamp to the last line, differ from it there and nowhere else): no defined result to match
        auto asym = [](const SwsVec *v) { if (!v) return false; for (int i = 0; i < v->length / 2; i++) if (v->coeff[i] != v->coeff[v->length - 1 - i]) return true; return false; };
        if (asym(sf.lumV) || asym(sf.chrV)) { set_error_msg("sws_getContext_cuda", "asymmetric vertical SwsFilter vectors are not taken over"); return nullptr; }
    }
    if (usesFilter && (srcRgb || srcYuy || src32 || srcPal || srcNV || D->pk422 || dstNV || D->bits != 8)) {
        set_error_msg("sws_getContext_cuda", "SwsFilter vectors are taken over for planar 8-bit yuv sources to packed rgb / planar 8-bit yuv destinations only");
        return nullptr;
    }
    // swscale.c:748-765: a yuv destination of the other range gets lum / chrRangeFromJpeg_c (1) or ...ToJpeg_c (2) between the two passes,
    // and none of the unscaled special converters (utils.c:1043-1044)
    const int rangeConv = (srcRange != dstRange && (planar || D->pk422)) ? (srcRange ? 1 : 2) : 0;
    if (rangeConv && D->bits == 16) {       // (the *Range*16_c variants work on the 19-bit lines that only exist in the tile kernel)
        set_error_msg("sws_getContext_cuda", "range conversion (full-range yuvj <-> limited-range yuv) to a 16-bit destination is not taken over");
        return nullptr;
    }
    if (srcBits > 8) {
        const char *why = nullptr;
        if (usesFilter) why = "SwsFilter vectors with a 9 / 10 / 16-bit source are not taken over";
        else if (rangeConv) why = "range conversion from a 9 / 10 / 16-bit source is not taken over";
        else if (planar && D->bits == 16) why = "9 / 10 / 16-bit source to a 16-bit destination (hScale16To19_c lines) is not taken over";
        // same size and sub-sampling, planar destination: planarCopyWrapper with its own depth conversions (swscale_unscaled.c:793-1020)
        else if (planar && !dstNV && unscaled && hs == D->hs && vs == D->vs)
            why = "9 / 10 / 16-bit source to a planar destination of the same size and sub-sampling is the reference's planarCopyWrapper: not taken over";
        if (why) { set_error_msg("sws_getContext_cuda", why); return nullptr; }
    }
    if (!rgb) flags &= ~SWS_FULL_CHR_H_INT;                 // only packed RGB knows the flag (utils.c:998-1014)
    SwsCudaContext *c = new (std::nothrow) SwsCudaContext();
    if (!c) return nullptr;
    c->srcFmt = srcIn; c->dstFmt = dstIn; c->S = S; c->D = D; c->rangeConv = rangeConv;
    double prm[2] = { param ? param[0] : SWS_PARAM_DEFAULT, param ? param[1] : SWS_PARAM_DEFAULT };
    if (derive_geometry(c->g, srcW, srcH, dstW, dstH, rgb, flags, &err, hs, vs, D->hs, D->vs)) goto fail;
    {
        const int fl = c->g.flags;
        const int lumFlags = (fl & SWS_BICUBLIN) ? (fl | SWS_BICUBIC) : fl;
        const int chrFlags = (fl & SWS_BICUBLIN) ? (fl | SWS_BILINEAR) : fl;
        if (design_filter(c->hLum, c->g.lumXInc, srcW, dstW, 1 << 14, lumFlags, prm, true, &err, sf.lumH, df.lumH)) goto fail;       // utils.c:1165-1198
        if (design_filter(c->hChr, c->g.chrXInc, c->g.chrSrcW, c->g.chrDstW, 1 << 14, chrFlags, prm, true, &err, sf.chrH, df.chrH)) goto fail;
        if (design_filter(c->vLum, c->g.lumYInc, srcH, dstH, 1 << 12, lumFlags, prm, false, &err, sf.lumV, df.lumV)) goto fail;
        if (design_filter(c->vChr, c->g.chrYInc, c->g.chrSrcH, c->g.chrDstH, 1 << 12, chrFlags, prm, false, &err, sf.chrV, df.chrV)) goto fail;
    }
    {
        static const int itu601[4] = { 104597, 132201, 25675, 53279 };     // ff_yuv2rgb_coeffs[SWS_CS_DEFAULT]
        rgb_constants(c->k, itu601, srcRange, 0, 1 << 16, 1 << 16);      // sws_getContext defaults, utils.c:1366-1368
        c->srcRange = srcRange;
    }
    c->route = choose_route(c, flags, unscaled, usesFilter, grayPal, rgb2rgb);
    if (c->route == R_FUSED && !(dstW & 15) && !(dstH & 1)) {
        bool ok = true;
        for (int y = 0; y < dstH && ok; y += 2) {
            const int f0 = c->vChr.pos[y] > -3 ? c->vChr.pos[y] : -3, f1 = c->vChr.pos[y + 1] > -3 ? c->vChr.pos[y + 1] : -3;
            if (f1 - f0 != 0 && f1 - f0 != 1) ok = false;       // the pair's windows must start at most one line apart
            for (int r = 0; r < 2 && ok; r++) {
                int lo = 2048, hi = 2048;
                for (int j = 0; j < 4; j++) { int k = c->vChr.coef[(size_t)(y + r) * 4 + j]; if (k < 0) lo += 255 * k; else hi += 255 * k; }
                if ((lo >> 12) <= -256 || (hi >> 12) >= 512) ok = false;
            }
        }
        c->fast_ok = ok;
    }
    if (!device_side) return c;
    if (upload_tables(c)) { destroy(c); return nullptr; }
    if (srcPal && cudaMalloc(&c->d_pal, 1024) != cudaSuccess) { set_error("sws_getContext_cuda", cudaGetLastError()); destroy(c); return nullptr; }
    if (gray) {
        c->grayPitch = (c->g.chrDstW + 63) & ~31;
        for (int k = 0; k < 2; k++)
            if (cudaMalloc(&c->d_gray[k], (size_t)c->grayPitch * (c->g.chrDstH + 2)) != cudaSuccess) { set_error("sws_getContext_cuda", cudaGetLastError()); destroy(c); return nullptr; }
    }
    if (c->fast_ok) {
        std::vector<SwsPairTaps> pt(dstH / 2);
        for (int rp = 0; rp < dstH / 2; rp++) {
            const int y = 2 * rp;
            const int f0 = c->vChr.pos[y] > -3 ? c->vChr.pos[y] : -3, f1 = c->vChr.pos[y + 1] > -3 ? c->vChr.pos[y + 1] : -3, d1 = f1 - f0;
            int k0[4], k1[5] = { 0, 0, 0, 0, 0 };
            for (int j = 0; j < 4; j++) { k0[j] = c->vChr.coef[(size_t)y * 4 + j]; k1[j + d1] = c->vChr.coef[(size_t)(y + 1) * 4 + j]; }
            SwsPairTaps t = {};
            for (int j = 0; j < 4; j++) {
                t.lo0 |= (uint32_t)(k0[j] & 255) << (8 * j); t.hi0 |= (uint32_t)((k0[j] >> 8) & 255) << (8 * j);
                t.lo1 |= (uint32_t)(k1[j] & 255) << (8 * j); t.hi1 |= (uint32_t)((k1[j] >> 8) & 255) << (8 * j);
                if ((k0[j] >> 8) < -128 || (k0[j] >> 8) > 127 || (k1[j] >> 8) < -128 || (k1[j] >> 8) > 127) c->fast_ok = false;
            }
            t.tap4 = k1[4]; t.first = f0;
            pt[rp] = t;
        }
        if (c->fast_ok && upload(&c->d_pair_taps, pt.data(), pt.size() * sizeof(SwsPairTaps))) { destroy(c); return nullptr; }
    }
    if (c->fast_ok) {            // the TMA kernel's table: per pair the int16 tap pairs of both rows, per four-pair tile its chroma line window
        const int pairs = dstH / 2, chrH = c->g.chrSrcH;
        std::vector<SwsPairTapsT> pt(pairs);
        bool ok = true;
        for (int rp = 0; rp < pairs; rp++) {
            SwsPairTapsT &t = pt[rp];
            const int16_t *k0 = &c->vChr.coef[(size_t)(2 * rp) * 4], *k1 = k0 + 4;
            t.k01_0 = (uint16_t)k0[0] | (uint32_t)(uint16_t)k0[1] << 16; t.k23_0 = (uint16_t)k0[2] | (uint32_t)(uint16_t)k0[3] << 16;
            t.k01_1 = (uint16_t)k1[0] | (uint32_t)(uint16_t)k1[1] << 16; t.k23_1 = (uint16_t)k1[2] | (uint32_t)(uint16_t)k1[3] << 16;
            t.first0 = c->vChr.pos[2 * rp] > -3 ? c->vChr.pos[2 * rp] : -3;
            t.first1 = c->vChr.pos[2 * rp + 1] > -3 ? c->vChr.pos[2 * rp + 1] : -3;
        }
        auto clampl = [&](int l) { return l < 0 ? 0 : l > chrH - 1 ? chrH - 1 : l; };
        for (int t0 = 0; t0 < pairs && ok; t0 += 4) {
            const int t1 = std::min(t0 + 4, pairs);
            int lo = INT_MAX, hi = INT_MIN;
            for (int rp = t0; rp < t1; rp++)
                for (int r = 0; r < 2; r++) {
                    const int f = r ? pt[rp].first1 : pt[rp].first0;
                    lo = std::min(lo, clampl(f)); hi = std::max(hi, clampl(f + 3));
                }
            if (hi - lo > 7) ok = false;
            bool interior = t1 - t0 == 4 && lo + 7 <= chrH - 1;
            for (int rp = t0; rp < t1 && interior; rp++) interior = pt[rp].first0 == lo + (rp - t0) && pt[rp].first1 == pt[rp].first0 + 1;
            for (int rp = t0; rp < t1; rp++) { pt[rp].base = lo; pt[rp].interior = interior; }
        }
        if (ok && pairs > 0) {
            static const int zero4[4] = { 0, 0, 0, 0 };
            if (upload(&c->d_pair_taps_t, pt.data(), pt.size() * sizeof(SwsPairTapsT)) || upload((void **)&c->d_tickets, zero4, sizeof(zero4))) {
                destroy(c); return nullptr;
            }
            c->tma_ok = true;
        }
    }
    if (c->route == R_SCALE) {
        int lr = 0, cr = 0, lo, hi;
        std::vector<int2> win;
        for (int y0 = 0; y0 < dstH; y0 += GT_H) {
            tile_line_window(c->vLum.pos.data(), c->vLum.size, y0, std::min(y0 + GT_H, dstH) - 1, srcH, lo, hi);
            lr = std::max(lr, hi - lo + 1); win.push_back(make_int2(lo, hi - lo + 1));
        }
        const size_t nLumWin = win.size();
        // vChr has chrDstH entries: dstH of them for packed rgb (no vertical chroma sub-sampling on that side)
        for (int y0 = 0; y0 < c->g.chrDstH; y0 += GT_H) {
            tile_line_window(c->vChr.pos.data(), c->vChr.size, y0, std::min(y0 + GT_H, c->g.chrDstH) - 1, c->g.chrSrcH, lo, hi);
            cr = std::max(cr, hi - lo + 1); win.push_back(make_int2(lo, hi - lo + 1));
        }
        const bool fullc = rgb && (flags & SWS_FULL_CHR_H_INT);
        const size_t need = rgb ? ((size_t)lr * GT_LW + (size_t)cr * (fullc ? 2 * GT_LW : GT_W)) * 4 : (size_t)std::max(lr, cr) * GT_LW * 4;
        if (need <= 96 * 1024 && !D->pk422 && !D->rgb16 && !rangeConv && srcBits == 8 && !srcGray) {          // (the packed 4:2:2 / 16-bpp output stages and the range conversion only exist in the two-pass path so far)
            c->tileLumRows = lr; c->tileChrRows = cr;
            if (upload((void **)&c->d_tile_win, win.data(), win.size() * sizeof(int2))) { destroy(c); return nullptr; }
            c->tileChrWinOff = nLumWin;
        }
        if (D->bits == 16 && !c->tileLumRows) {      // the two-pass fallback keeps 15-bit lines in int16 planes
            set_error_msg("sws_getContext_cuda", "16-bit destination: the vertical filter window does not fit in shared memory (19-bit lines exist only there)");
            destroy(c); return nullptr;
        }
        c->lumStridePx = (dstW + 1 + 7) & ~7;          // multiples of 8 samples: 16-byte aligned rows for the vector passes
        c->chrStridePx = (c->g.chrDstW + 7) & ~7;
        if (cudaMalloc(&c->d_lum, (size_t)c->lumStridePx * srcH * 2) != cudaSuccess ||
            cudaMalloc(&c->d_chrU, (size_t)c->chrStridePx * c->g.chrSrcH * 2) != cudaSuccess ||
            cudaMalloc(&c->d_chrV, (size_t)c->chrStridePx * c->g.chrSrcH * 2) != cudaSuccess) {
            set_error("sws_getContext_cuda", cudaGetLastError());
            destroy(c); return nullptr;
        }
    }
    return c;
fail:
    set_error_msg("sws_getContext_cuda", err ? err : "init failed");
    delete c;
    return nullptr;
}

// ---------------------------------------------------------------------------------------------------
// what a context reads and writes
// ---------------------------------------------------------------------------------------------------
// The planes of a picture as the caller lays them out: how many, the bytes of a row's pixels, the rows
struct PlaneGeom { int n; size_t row[3]; int rows[3]; };
static PlaneGeom src_planes(const SwsCudaContext *c)
{
    const SwsGeometry &g = c->g;
    if (is_packed_src(c->S)) return { 1, { (size_t)g.srcW * c->S->bpp, 0, 0 }, { g.srcH, 0, 0 } };
    const size_t s = c->srcFmt->bits > 8 ? 2 : 1, nv = c->S->fam == FAM_NV;
    return { nv ? 2 : 3, { g.srcW * s, g.chrSrcW * (nv ? 2 : 1) * s, g.chrSrcW * s }, { g.srcH, g.chrSrcH, g.chrSrcH } };
}
static PlaneGeom dst_planes(const SwsCudaContext *c)
{
    const SwsGeometry &g = c->g;
    if (!is_planar(c->D)) return { 1, { (size_t)g.dstW * c->D->bpp, 0, 0 }, { g.dstH, 0, 0 } };
    const size_t s = c->D->bits > 8 ? 2 : 1, nv = c->D->fam == FAM_NV;
    return { nv ? 2 : 3, { g.dstW * s, g.chrDstW * (nv ? 2 : 1) * s, g.chrDstW * s }, { g.dstH, g.chrDstH, g.chrDstH } };
}

// The planar -> packed 4:2:2 converters' pair count over a row of width w: the reference's 64-bit loop converts two pairs per step
// (rgb2rgb_template.c:374-386), so an odd pair count is rounded up and the extra pair reads / writes past the nominal width --
// reproduced when every row involved has room for it
static int to422_pairs(int w, int dstStride, const int srcStride[3])
{
    const int pairs = w >> 1, pairs_r = (pairs + 1) & ~1;
    return pairs_r > pairs && dstStride >= 4 * pairs_r && srcStride[0] >= 2 * pairs_r && srcStride[1] >= pairs_r && srcStride[2] >= pairs_r ? pairs_r : pairs;
}

// The pixels of each packed destination row the route writes
static int packed_cols(const SwsCudaContext *c, int dstStride, const int srcStride[3])
{
    const int w = c->g.dstW;
    switch (c->route) {
    case R_TABLE: return w & ~1;                            // the unscaled table converter leaves an odd last column alone
    case R_422_FROM_422P: case R_422_FROM_420P: return 2 * to422_pairs(w, dstStride, srcStride);
    case R_SCALE: case R_FUSED: case R_RGB48:               // whole pixel pairs, one pixel past an odd width when the row has room; single
        return (w & 1) && !c->dev.full && dstStride >= (w + 1) * c->D->bpp ? w + 1 : w;        // pixels with SWS_FULL_CHR_H_INT
    default: return w;
    }
}

// The samples of each planar destination plane the route writes: luma columns; chroma columns and rows
static void planar_extent(const SwsCudaContext *c, int &w, int &cw, int &ch)
{
    const SwsGeometry &g = c->g;
    const bool nvSplit = c->route == R_COPY && c->S->fam == FAM_NV;
    w = c->route == R_BGR24_YV12 ? g.dstW & ~1 : g.dstW;     // rgb24toyv12_c converts whole pixel pairs only
    // nv12ToPlanarWrapper and planarToNv12Wrapper move srcW / 2 x srcH / 2 chroma samples: an odd last column / row stays untouched;
    // the packed -> yuv420p converters write srcH / 2 chroma rows
    cw = nvSplit || c->route == R_BGR24_YV12 || c->route == R_NV_INTERLEAVE ? g.srcW / 2 : g.chrDstW;
    ch = nvSplit || c->route == R_BGR24_YV12 || c->route == R_YUYV_420P || c->route == R_NV_INTERLEAVE ? g.srcH / 2 : g.chrDstH;
}

// ---------------------------------------------------------------------------------------------------
// dispatch
// ---------------------------------------------------------------------------------------------------
static FusedArgs fused_args(const uint8_t *const src[3], const int srcStride[3], const size_t srcFrame[3], uint8_t *dst, int dstStride, size_t dstFrame)
{
    FusedArgs a;
    a.y = src[0]; a.u = src[1]; a.v = src[2]; a.dst = dst;
    a.yStride = srcStride[0]; a.uStride = srcStride[1]; a.vStride = srcStride[2]; a.dstStride = dstStride;
    a.yFrame = srcFrame[0]; a.uFrame = srcFrame[1]; a.vFrame = srcFrame[2]; a.dstFrame = dstFrame;
    return a;
}

// the interior fast path of the fused same-size kernel over row pairs [a.rp0, a.rp1): TMA-staged (sws_fused_tma.cu) when tensor maps can
// describe the planes, else the LDG kernel
static int launch_fused_fast(SwsCudaContext *c, const FusedArgs &a, int nframes, cudaStream_t st)
{
    const SwsDev &p = c->dev;
#ifndef AVB_HOSTSIM
    if (c->tma_ok) {
        int slot = 0;               // the counter of the stream (SwsCudaContext::d_tickets)
        for (int i = 0; i < 3; i++) if (c->streams_ok && st == c->streams[i]) slot = 1 + i;
        const int r = sws_fused_tma_launch(p.k, p.bgr, p.dstW, p.dstH, p.chrSrcW, p.chrSrcH, a, (const SwsPairTapsT *)c->d_pair_taps_t,
                                           c->d_tickets + slot, nframes, st);
        if (r <= 0) return r;
    }
#endif
    const int rp1 = a.rp1 < p.dstH / 2 ? a.rp1 : p.dstH / 2;
    if (rp1 <= a.rp0) return 0;
    dim3 b2(32, 4), g2((p.dstW / 16 + 31) / 32, (rp1 - a.rp0 + 3) / 4, nframes);
    FusedArgs a2 = a; a2.rp1 = rp1;
    const SwsPairTaps *pt = (const SwsPairTaps *)c->d_pair_taps;
    if (p.bgr) sws_fused_rgb24_v3_kernel<true><<<g2, b2, 0, st>>>(p, a2, pt); else sws_fused_rgb24_v3_kernel<false><<<g2, b2, 0, st>>>(p, a2, pt);
    return check_launch("sws_scale:fused");
}

static int run_fused(SwsCudaContext *c, const uint8_t *const src[3], const int srcStride[3], const size_t srcFrame[3],
                     uint8_t *const dst[3], const int dstStride[3], const size_t dstFrame[3], int nframes, cudaStream_t st)
{
    const SwsDev &p = c->dev;
    FusedArgs a = fused_args(src, srcStride, srcFrame, dst[0], dstStride[0], dstFrame[0]);
    // vector accesses need 8-byte aligned luma / output rows and 4-byte aligned chroma rows
    bool aligned = !((uintptr_t)a.y & 7) && !(a.yStride & 7) && !((uintptr_t)a.dst & 7) && !(a.dstStride & 7) && !(a.yFrame & 7) &&
                   !(a.dstFrame & 7) && !((uintptr_t)a.u & 3) && !((uintptr_t)a.v & 3) && !(a.uStride & 3) && !(a.vStride & 3) &&
                   !(a.uFrame & 3) && !(a.vFrame & 3);
    const bool a16 = aligned && !((uintptr_t)a.y & 15) && !(a.yStride & 15) && !((uintptr_t)a.dst & 15) && !(a.dstStride & 15) &&
                     !(a.yFrame & 15) && !(a.dstFrame & 15) && !((uintptr_t)a.u & 7) && !((uintptr_t)a.v & 7) && !(a.uStride & 7) &&
                     !(a.vStride & 7) && !(a.uFrame & 7) && !(a.vFrame & 7) && !((uintptr_t)p.vChrF & 15);
    if (c->fast_ok && a16) {
        a.rp0 = 0; a.rp1 = p.dstH / 2;
        return launch_fused_fast(c, a, nframes, st);
    }
    dim3 b(32, 8), g((p.dstW + 255) / 256, (p.dstH + 15) / 16, nframes);
    if (aligned) sws_fused_rgb24_kernel<true><<<g, b, 0, st>>>(p, a);
    else         sws_fused_rgb24_kernel<false><<<g, b, 0, st>>>(p, a);    // same arithmetic, byte accesses
    return check_launch("sws_scale:fused");
}

// the general scaler: fused per output tile when the vertical windows fit in shared memory, else two passes over line planes
static int run_scale(SwsCudaContext *c, const uint8_t *const src[3], const int srcStride[3], const size_t srcFrame[3],
                     uint8_t *const dst[3], const int dstStride[3], const size_t dstFrame[3], int nframes, cudaStream_t st)
{
    const SwsDev &p = c->dev;
    const bool planar = is_planar(c->D);
    if (c->tileLumRows && (tuning("sws_general_variant") != 1 || p.dstBits == 16)) {       // general path, fused per output tile
        TileArgs a;
        a.y = src[0]; a.u = src[1]; a.v = src[2]; a.dst0 = dst[0]; a.dst1 = dst[1]; a.dst2 = dst[2];
        a.yStride = srcStride[0]; a.uStride = srcStride[1]; a.vStride = srcStride[2];
        a.yFrame = srcFrame[0]; a.uFrame = srcFrame[1]; a.vFrame = srcFrame[2];
        a.dstStride0 = dstStride[0]; a.dstFrame0 = dstFrame[0];
        a.dstStride1 = planar ? dstStride[1] : 0; a.dstStride2 = planar ? dstStride[2] : 0;
        a.dstFrame1 = planar ? dstFrame[1] : 0; a.dstFrame2 = planar ? dstFrame[2] : 0;
        a.lumRows = c->tileLumRows; a.chrRows = c->tileChrRows;
        a.lumWin = c->d_tile_win; a.chrWin = c->d_tile_win + c->tileChrWinOff;
        a.lumXInc = c->g.lumXInc; a.chrXInc = c->g.chrXInc;
        a.vec = !((uintptr_t)a.dst0 & 7) && !(a.dstStride0 & 7) && !(a.dstFrame0 & 7);
        // (the fast-bilinear line functions only exist for 15-bit lines: a 16-bit destination gets the designed filter, swscale.c:728-741)
        const bool fastb = (c->g.flags & SWS_FAST_BILINEAR) && p.dstBits != 16;
        const int fsl = fastb ? -1 : p.hLumSize, fsc = fastb ? -1 : p.hChrSize;
        const dim3 gl((p.dstW + GT_W - 1) / GT_W, (p.dstH + GT_H - 1) / GT_H, nframes);
        if (!planar) {
            const size_t smem = ((size_t)a.lumRows * GT_LW + (size_t)a.chrRows * (p.full ? 2 * GT_LW : GT_W)) * 4;
            auto go = [&](auto kern) {
                cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, 96 * 1024);
                kern<<<gl, GT_THREADS, smem, st>>>(p, a);
            };
            if (p.full) {
                if (fsl == -1)                 go(sws_tile_rgb24_kernel<-1, -1, true>);
                else if (fsl == 4 && fsc == 4) go(sws_tile_rgb24_kernel<4, 4, true>);
                else if (fsl == 8 && fsc == 8) go(sws_tile_rgb24_kernel<8, 8, true>);
                else                           go(sws_tile_rgb24_kernel<0, 0, true>);
            }
            else if (fsl == -1)             go(sws_tile_rgb24_kernel<-1, -1>);
            else if (fsl == 2 && fsc == 2)  go(sws_tile_rgb24_kernel<2, 2>);
            else if (fsl == 4 && fsc == 4)  go(sws_tile_rgb24_kernel<4, 4>);
            else if (fsl == 8 && fsc == 8)  go(sws_tile_rgb24_kernel<8, 8>);
            else                            go(sws_tile_rgb24_kernel<0, 0>);
        } else {
            const dim3 gc((p.chrDstW + GT_W - 1) / GT_W, (p.chrDstH + GT_H - 1) / GT_H, 2 * nframes);
            auto go = [&](auto kl, auto kc) {
                cudaFuncSetAttribute(kl, cudaFuncAttributeMaxDynamicSharedMemorySize, 96 * 1024);
                cudaFuncSetAttribute(kc, cudaFuncAttributeMaxDynamicSharedMemorySize, 96 * 1024);
                kl<<<gl, GT_THREADS, (size_t)a.lumRows * GT_LW * 4, st>>>(p, a);
                kc<<<gc, GT_THREADS, (size_t)a.chrRows * GT_LW * 4, st>>>(p, a);
            };
            if (fsl == -1)                  go(sws_tile_plane_kernel<-1, false>, sws_tile_plane_kernel<-1, true>);
            else if (fsl == 2 && fsc == 2)  go(sws_tile_plane_kernel<2, false>, sws_tile_plane_kernel<2, true>);
            else if (fsl == 4 && fsc == 4)  go(sws_tile_plane_kernel<4, false>, sws_tile_plane_kernel<4, true>);
            else if (fsl == 8 && fsc == 8)  go(sws_tile_plane_kernel<8, false>, sws_tile_plane_kernel<8, true>);
            else                            go(sws_tile_plane_kernel<0, false>, sws_tile_plane_kernel<0, true>);
        }
        return check_launch("sws_scale:tile");
    }
    for (int f = 0; f < nframes; f++) {      // general path, two passes: frames are serialised on the stream (shared line planes)
        const uint8_t *y = src[0] + f * srcFrame[0], *u = src[1] + f * srcFrame[1], *v = src[2] + f * srcFrame[2];
        dim3 b(256);
        if (p.srcGray) {                     // luma only; the chroma lines keep the bytes of 64 sws_init_context wrote (0x4040 per 15-bit sample)
            if (c->g.flags & SWS_FAST_BILINEAR)
                sws_hscale_fast_kernel<<<dim3((p.dstW + 255) / 256, p.srcH), b, 0, st>>>(y, srcStride[0], c->d_lum, c->lumStridePx, p.srcW, p.dstW, p.srcH, c->g.lumXInc, 0);
            else
                sws_hscale8to15_x4_kernel<<<dim3((p.dstW + 1023) / 1024, p.srcH), b, 0, st>>>(y, srcStride[0], c->d_lum, c->lumStridePx, p.hLumF, p.hLumP, p.hLumSize, p.dstW, p.srcH);
            AVB_CUDA(cudaMemsetAsync(c->d_chrU, 0x40, (size_t)c->chrStridePx * p.chrSrcH * 2, st), "sws_scale:gray8");
            AVB_CUDA(cudaMemsetAsync(c->d_chrV, 0x40, (size_t)c->chrStridePx * p.chrSrcH * 2, st), "sws_scale:gray8");
        } else if (p.srcBits > 8) {                  // no fast-bilinear line functions for these sources (swscale.c:733-743): the designed bank
            sws_hscale16to15_kernel<<<dim3((p.dstW + 255) / 256, p.srcH), b, 0, st>>>(y, srcStride[0], c->d_lum, c->lumStridePx, p.hLumF, p.hLumP, p.hLumSize, p.dstW, p.srcH, p.srcBits, p.srcBE);
            sws_hscale16to15_kernel<<<dim3((p.chrDstW + 255) / 256, p.chrSrcH), b, 0, st>>>(u, srcStride[1], c->d_chrU, c->chrStridePx, p.hChrF, p.hChrP, p.hChrSize, p.chrDstW, p.chrSrcH, p.srcBits, p.srcBE);
            sws_hscale16to15_kernel<<<dim3((p.chrDstW + 255) / 256, p.chrSrcH), b, 0, st>>>(v, srcStride[2], c->d_chrV, c->chrStridePx, p.hChrF, p.hChrP, p.hChrSize, p.chrDstW, p.chrSrcH, p.srcBits, p.srcBE);
        } else if (c->g.flags & SWS_FAST_BILINEAR) {
            sws_hscale_fast_kernel<<<dim3((p.dstW + 255) / 256, p.srcH), b, 0, st>>>(y, srcStride[0], c->d_lum, c->lumStridePx, p.srcW, p.dstW, p.srcH, c->g.lumXInc, 0);
            sws_hscale_fast_kernel<<<dim3((p.chrDstW + 255) / 256, p.chrSrcH), b, 0, st>>>(u, srcStride[1], c->d_chrU, c->chrStridePx, p.chrSrcW, p.chrDstW, p.chrSrcH, c->g.chrXInc, 1);
            sws_hscale_fast_kernel<<<dim3((p.chrDstW + 255) / 256, p.chrSrcH), b, 0, st>>>(v, srcStride[2], c->d_chrV, c->chrStridePx, p.chrSrcW, p.chrDstW, p.chrSrcH, c->g.chrXInc, 1);
        } else {
            sws_hscale8to15_x4_kernel<<<dim3((p.dstW + 1023) / 1024, p.srcH), b, 0, st>>>(y, srcStride[0], c->d_lum, c->lumStridePx, p.hLumF, p.hLumP, p.hLumSize, p.dstW, p.srcH);
            sws_hscale8to15_x4_kernel<<<dim3((p.chrDstW + 1023) / 1024, p.chrSrcH), b, 0, st>>>(u, srcStride[1], c->d_chrU, c->chrStridePx, p.hChrF, p.hChrP, p.hChrSize, p.chrDstW, p.chrSrcH);
            sws_hscale8to15_x4_kernel<<<dim3((p.chrDstW + 1023) / 1024, p.chrSrcH), b, 0, st>>>(v, srcStride[2], c->d_chrV, c->chrStridePx, p.hChrF, p.hChrP, p.hChrSize, p.chrDstW, p.chrSrcH);
        }
        if (c->rangeConv) {                 // hyscale() / hcscale() call c->lumConvertRange / chrConvertRange on every converted line (swscale.c:223-225, 270-272)
            if (sws_launch_range(c->d_lum, c->lumStridePx, p.dstW, p.srcH, c->rangeConv == 1 ? 0 : 2, st) ||
                sws_launch_range(c->d_chrU, c->chrStridePx, p.chrDstW, p.chrSrcH, c->rangeConv == 1 ? 1 : 3, st) ||
                sws_launch_range(c->d_chrV, c->chrStridePx, p.chrDstW, p.chrSrcH, c->rangeConv == 1 ? 1 : 3, st)) return -1;
        }
        if (planar) {
            sws_vscale_plane_kernel<<<dim3((p.dstW + 255) / 256, p.dstH), b, 0, st>>>(c->d_lum, c->lumStridePx, p.srcH, p.vLumF, p.vLumP, p.vLumSize, dst[0] + f * dstFrame[0], dstStride[0], p.dstW, p.dstH, p.dstBits, p.dstBE, 1, p.dither, 0);
            sws_vscale_plane_kernel<<<dim3((p.chrDstW + 255) / 256, p.chrDstH), b, 0, st>>>(c->d_chrU, c->chrStridePx, p.chrSrcH, p.vChrF, p.vChrP, p.vChrSize, dst[1] + f * dstFrame[1], dstStride[1], p.chrDstW, p.chrDstH, p.dstBits, p.dstBE, p.chrStep, p.dither, 0);
            sws_vscale_plane_kernel<<<dim3((p.chrDstW + 255) / 256, p.chrDstH), b, 0, st>>>(c->d_chrV, c->chrStridePx, p.chrSrcH, p.vChrF, p.vChrP, p.vChrSize, dst[2] + f * dstFrame[2], dstStride[2], p.chrDstW, p.chrDstH, p.dstBits, p.dstBE, p.chrStep, p.dither, 3);      // chrDither8 with offset 3 for V (swscale.c:636-644)
        } else {
            int pairs = (p.dstW + 1) >> 1;
            uint8_t *d0 = dst[0] + f * dstFrame[0];
            const bool x_path = !((p.vLumSize == 1 && p.vChrSize <= 2) || (p.vLumSize == 2 && p.vChrSize == 2));
            if (p.pk422 || p.rgb16)
                sws_vscale_rgb24_kernel<<<dim3((pairs + 255) / 256, p.dstH), b, 0, st>>>(p, c->d_lum, c->d_chrU, c->d_chrV, c->lumStridePx, c->chrStridePx, d0, dstStride[0]);
            else if (p.full)
                sws_vscale_rgb24_full_kernel<<<dim3((p.dstW + 255) / 256, p.dstH), b, 0, st>>>(p, c->d_lum, c->d_chrU, c->d_chrV, c->lumStridePx, c->chrStridePx, d0, dstStride[0]);
            else if (x_path && !(p.dstW & 7) && !(dstStride[0] & 7) && !((uintptr_t)d0 & 7))
                sws_vscale_rgb24_x8_kernel<<<dim3((p.dstW / 8 + 127) / 128, p.dstH), 128, 0, st>>>(p, c->d_lum, c->d_chrU, c->d_chrV, c->lumStridePx, c->chrStridePx, d0, dstStride[0]);
            else
                sws_vscale_rgb24_kernel<<<dim3((pairs + 255) / 256, p.dstH), b, 0, st>>>(p, c->d_lum, c->d_chrU, c->d_chrV, c->lumStridePx, c->chrStridePx, d0, dstStride[0]);
        }
        if (check_launch("sws_scale:general")) return -1;
    }
    return 0;
}

// byte map of sws_rgb_map_kernel / sws_pal8_rgb_kernel: destination byte i of a pixel takes source byte (map >> 4 i) & 15, 15 = 255.
// from[] holds the source byte of r, g, b and a (-1: none)
static unsigned channel_map(const PixFmt *d, const int (&from)[4])
{
    const int to[4] = { d->r, d->g, d->b, d->a };
    unsigned map = 0;
    for (int ch = 0; ch < 4; ch++) if (to[ch] >= 0) map |= (unsigned)(from[ch] >= 0 ? from[ch] : 15) << (4 * to[ch]);
    return map;
}

// One batch of frames on device pointers: the source pre-pass, the route, the 32-bit expansion.  src[] / dst[] are the planes the
// route reads and writes (for gray8 the public entry points substituted them).
static int run_frames(SwsCudaContext *c, const uint8_t *const src_[3], const int srcStride_[3], const size_t srcFrame_[3],
                      uint8_t *const dst_[3], const int dstStride_[3], const size_t dstFrame_[3], int nframes, cudaStream_t st)
{
    if (nframes <= 0) return 0;
    const SwsDev &p = c->dev;
    const PixFmt *S = c->S, *D = c->D;
    const Route r = c->route;
    const int w = p.srcW, h = p.srcH;
    const uint8_t *src[3] = { src_[0], src_[1], src_[2] };
    int srcStride[3] = { srcStride_[0], srcStride_[1], srcStride_[2] };
    size_t srcFrame[3] = { srcFrame_[0], srcFrame_[1], srcFrame_[2] };
    uint8_t *dst[3] = { dst_[0], dst_[1], dst_[2] };
    int dstStride[3] = { dstStride_[0], dstStride_[1], dstStride_[2] };
    size_t dstFrame[3] = { dstFrame_[0], dstFrame_[1], dstFrame_[2] };
    if (D->fam == FAM_NV && r != R_NV_INTERLEAVE) {      // U and V are the even / odd bytes of plane 1 (chrStep 2 in the kernels)
        const int v = D->fmt == PIX_NV21;
        dst[2] = dst_[1] + (v ? 0 : 1); dst[1] = dst_[1] + v;
        dstStride[2] = dstStride[1]; dstFrame[2] = dstFrame[1];
    }
    // 32-bit rgb destinations: the rgb24 pipeline into a scratch picture, then one expansion pass (+ 6 B per pixel of traffic; fusing the
    // 4-byte store into every output kernel is the next step for this format family)
    const bool expand = D->fam == FAM_RGB32 && ROUTES[r].planar;
    const int pitch32 = ((p.dstW + 1) * 3 + 15) & ~15;
    const size_t frame32 = (size_t)pitch32 * p.dstH;
    if (expand) {
        if (grow(c->d_rgb, c->rgb_bytes, frame32 * nframes, st, "sws_scale:rgb32")) return -1;
        dst[0] = c->d_rgb; dst[1] = dst[2] = nullptr;
        dstStride[0] = pitch32; dstStride[1] = dstStride[2] = 0;
        dstFrame[0] = frame32; dstFrame[1] = dstFrame[2] = 0;
    }
    if (ROUTES[r].planar && S->fam == FAM_NV) {      // semi-planar sources: split the interleaved chroma plane (input.c:475-497)
        const int pitch = (p.chrSrcW + 15) & ~15, swap = S->fmt == PIX_NV21;
        const size_t plane = (size_t)pitch * p.chrSrcH;
        if (grow(c->d_nv, c->nv_bytes, 2 * plane * nframes, st, "sws_scale:nv12")) return -1;
        uint8_t *U = c->d_nv, *V = c->d_nv + plane * nframes;
        sws_split_nv_kernel<<<dim3((p.chrSrcW + 1023) / 1024, p.chrSrcH, nframes), 256, 0, st>>>(src[1], srcStride[1], srcFrame[1], swap ? V : U, swap ? U : V,
                                                                                              pitch, plane, plane, p.chrSrcW, p.chrSrcH);
        if (check_launch("sws_scale:nv12 split")) return -1;
        src[1] = U; src[2] = V; srcStride[1] = srcStride[2] = pitch; srcFrame[1] = srcFrame[2] = plane;
    } else if (ROUTES[r].planar && is_packed_src(S)) {
        // packed sources: the input readers (input.c) into planes, + srcW * srcH * (1 + 2 / 2^hs) bytes written and read again
        const int yPitch = (w + 15) & ~15, cPitch = (p.chrSrcW + 15) & ~15;
        const size_t yPlane = (size_t)yPitch * h, cPlane = (size_t)cPitch * p.chrSrcH;
        if (grow(c->d_nv, c->nv_bytes, (yPlane + 2 * cPlane) * nframes, st, "sws_scale:reader")) return -1;
        uint8_t *Y = c->d_nv, *U = Y + yPlane * nframes, *V = U + cPlane * nframes;
        const dim3 grid(((w + 1) / 2 + 255) / 256, h, nframes);
        const int half = p.chrSrcW != w;
        if (S->fam == FAM_PAL8) {
            if (!src[1]) { set_error_msg("sws_scale", "pal8 source without a palette in plane 1"); return -1; }
            sws_read_pal8_kernel<<<dim3((w + 255) / 256, h, nframes), 256, 0, st>>>(src[0], srcStride[0], srcFrame[0], src[1], srcFrame[1], Y, U, V, yPitch, yPlane, w, h);
        } else if (S->fam == FAM_RGB24) sws_read_packed_kernel<1><<<grid, 256, 0, st>>>(src[0], srcStride[0], srcFrame[0], Y, U, V, yPitch, cPitch, yPlane, cPlane, w, h, S->r, S->g, S->b, half);
        else if (S->fam == FAM_RGB32)   sws_read_packed_kernel<4><<<grid, 256, 0, st>>>(src[0], srcStride[0], srcFrame[0], Y, U, V, yPitch, cPitch, yPlane, cPlane, w, h, S->r, S->g, S->b, half);
        else if (S->pk422 == 1)         sws_read_packed_kernel<2><<<grid, 256, 0, st>>>(src[0], srcStride[0], srcFrame[0], Y, U, V, yPitch, cPitch, yPlane, cPlane, w, h, 0, 0, 0, 1);
        else                            sws_read_packed_kernel<3><<<grid, 256, 0, st>>>(src[0], srcStride[0], srcFrame[0], Y, U, V, yPitch, cPitch, yPlane, cPlane, w, h, 0, 0, 0, 1);
        if (check_launch("sws_scale:reader")) return -1;
        src[0] = Y; src[1] = U; src[2] = V;
        srcStride[0] = yPitch; srcStride[1] = srcStride[2] = cPitch;
        srcFrame[0] = yPlane; srcFrame[1] = srcFrame[2] = cPlane;
    }
    switch (r) {
    case R_PAL8_RGB: {             // the palette lookup of palToRgbWrapper
        if (!src[1]) { set_error_msg("sws_scale", "pal8 source without a palette in plane 1"); return -1; }
        sws_pal8_rgb_kernel<<<dim3((w + 255) / 256, h, nframes), 256, 0, st>>>(src[0], srcStride[0], srcFrame[0], src[1], srcFrame[1], dst[0], dstStride[0], dstFrame[0],
                                                                            w, h, D->bpp, channel_map(D, { 0, 1, 2, -1 }));
        return check_launch("sws_scale:pal8 -> rgb");
    }
    case R_GRAY_RGB:               // the pseudo-palette lookup is r = g = b = sample, alpha 255
        sws_rgb_map_kernel<<<dim3((w + 255) / 256, h, nframes), 256, 0, st>>>(src[0], srcStride[0], srcFrame[0], dst[0], dstStride[0], dstFrame[0], w, h, 1, D->bpp, channel_map(D, { 0, 0, 0, -1 }));
        return check_launch("sws_scale:gray8 -> rgb");
    case R_RGB_REMAP:
        sws_rgb_map_kernel<<<dim3((w + 255) / 256, h, nframes), 256, 0, st>>>(src[0], srcStride[0], srcFrame[0], dst[0], dstStride[0], dstFrame[0], w, h, S->bpp, D->bpp,
                                                                           channel_map(D, { S->r, S->g, S->b, S->a }));
        return check_launch("sws_scale:rgb2rgb");
    case R_RGB_COPY: case R_RGB24_SWAP:
        sws_rgb24_shuffle_kernel<<<dim3((w + 255) / 256, h, nframes), 256, 0, st>>>(src[0], srcStride[0], srcFrame[0], dst[0], dstStride[0], dstFrame[0], w, h, r == R_RGB24_SWAP);
        return check_launch("sws_scale:rgb24 shuffle");
    case R_BGR24_YV12: case R_YUYV_420P: case R_YUYV_422P:
        if (dstStride[1] != dstStride[2]) { set_error_msg("sws_scale", "packed -> yuv420p needs equal chroma pitches"); return -1; }
        if (r == R_YUYV_422P) {
            sws_yuyv_yuv422p_kernel<<<dim3(((w + 1) / 2 + 255) / 256, h, nframes), 256, 0, st>>>(src[0], srcStride[0], srcFrame[0], dst[0], dst[1], dst[2], dstStride[0], dstStride[1],
                                                                                            dstFrame[0], dstFrame[1], dstFrame[2], w, h, S->pk422 == 2);
        } else if (r == R_BGR24_YV12) {
            if (w >> 1) sws_bgr24_yv12_kernel<<<dim3(((w >> 1) + 255) / 256, h, nframes), 256, 0, st>>>(src[0], srcStride[0], srcFrame[0], dst[0], dst[1], dst[2], dstStride[0], dstStride[1],
                                                                                                    dstFrame[0], dstFrame[1], dstFrame[2], w, h);
        } else {
            sws_yuyv_yv12_kernel<<<dim3(((w + 1) / 2 + 255) / 256, h, nframes), 256, 0, st>>>(src[0], srcStride[0], srcFrame[0], dst[0], dst[1], dst[2], dstStride[0], dstStride[1],
                                                                                         dstFrame[0], dstFrame[1], dstFrame[2], w, h, S->pk422 == 2);
        }
        return check_launch("sws_scale:packed -> planar");
    case R_422_COPY:
        for (int f = 0; f < nframes; f++)
            AVB_CUDA(cudaMemcpy2DAsync(dst[0] + f * dstFrame[0], dstStride[0], src[0] + f * srcFrame[0], srcStride[0], (size_t)w * 2, h, cudaMemcpyDeviceToDevice, st), "sws_scale:copy");
        return 0;
    case R_422_FROM_422P: case R_422_FROM_420P: {
        if (srcStride[1] != srcStride[2]) { set_error_msg("sws_scale", "planar -> packed 4:2:2 needs equal chroma pitches"); return -1; }
        const int np = to422_pairs(w, dstStride[0], srcStride);
        if (np)
            sws_planar_to_422_kernel<<<dim3((np + 255) / 256, h, nframes), 256, 0, st>>>(src[0], srcStride[0], srcFrame[0], src[1], src[2], srcStride[1], srcFrame[1], srcFrame[2],
                                                                                      dst[0], dstStride[0], dstFrame[0], 2 * np, r == R_422_FROM_420P, D->pk422 == 2);
        return check_launch("sws_scale:planar -> packed 4:2:2");
    }
    case R_NV_INTERLEAVE: {
        for (int f = 0; f < nframes; f++)
            AVB_CUDA(cudaMemcpy2DAsync(dst[0] + f * dstFrame[0], dstStride[0], src[0] + f * srcFrame[0], srcStride[0], w, h, cudaMemcpyDeviceToDevice, st), "sws_scale:copy");
        const int u = D->fmt == PIX_NV21 ? 2 : 1, v = 3 - u;
        if (w / 2 > 0 && h / 2 > 0)
            sws_interleave_kernel<<<dim3((w / 2 + 255) / 256, h / 2, nframes), 256, 0, st>>>(src[u], srcStride[u], srcFrame[u], src[v], srcStride[v], srcFrame[v],
                                                                                         dst[1], dstStride[1], dstFrame[1], w / 2);
        return check_launch("sws_scale:planar -> nv12");
    }
    case R_COPY:
        if (S->fam == FAM_NV) {        // nv12ToPlanarWrapper (swscale_unscaled.c:160-181): luma copy + a split of srcW/2 x srcH/2 samples
            const int swap = S->fmt == PIX_NV21;
            for (int f = 0; f < nframes; f++)
                AVB_CUDA(cudaMemcpy2DAsync(dst[0] + f * dstFrame[0], dstStride[0], src[0] + f * srcFrame[0], srcStride[0], w, h, cudaMemcpyDeviceToDevice, st), "sws_scale:copy");
            if (w / 2 > 0 && h / 2 > 0) {
                if (dstStride[1] != dstStride[2]) { set_error_msg("sws_scale", "nv12 -> planar copy needs equal chroma pitches"); return -1; }
                sws_split_nv_kernel<<<dim3((w / 2 + 1023) / 1024, h / 2, nframes), 256, 0, st>>>(src[1], srcStride[1], srcFrame[1], dst[swap ? 2 : 1], dst[swap ? 1 : 2],
                                                                                             dstStride[1], dstFrame[swap ? 2 : 1], dstFrame[swap ? 1 : 2], w / 2, h / 2);
            }
            return check_launch("sws_scale:nv12 copy");
        }
        if (p.dstBits != 8) {
            for (int pl = 0; pl < 3; pl++) {
                const int pw = pl ? p.chrSrcW : w, ph = pl ? p.chrSrcH : h;
                sws_copy_plane_up_kernel<<<dim3((pw + 255) / 256, ph, nframes), 256, 0, st>>>(src[pl], srcStride[pl], srcFrame[pl], dst[pl], dstStride[pl], dstFrame[pl], pw, ph, p.dstBits - 8, p.dstBE);
            }
            return check_launch("sws_scale:copy");
        }
        for (int f = 0; f < nframes; f++)
            for (int pl = 0; pl < 3; pl++) {
                // a gray source: the luma plane, and 128 in the planes the source does not have (swscale_unscaled.c:812-823)
                if (pl && p.srcGray)
                    AVB_CUDA(cudaMemset2DAsync(dst[pl] + f * dstFrame[pl], dstStride[pl], 128, p.chrDstW, p.chrDstH, st), "sws_scale:copy");
                else
                    AVB_CUDA(cudaMemcpy2DAsync(dst[pl] + f * dstFrame[pl], dstStride[pl], src[pl] + f * srcFrame[pl], srcStride[pl], pl ? p.chrSrcW : w,
                                               pl ? p.chrSrcH : h, cudaMemcpyDeviceToDevice, st), "sws_scale:copy");
            }
        return 0;
    case R_TABLE: {
        FusedArgs a = fused_args(src, srcStride, srcFrame, dst[0], dstStride[0], dstFrame[0]);
        if (!S->vs) { a.uStride <<= 1; a.vStride <<= 1; }    // a 4:2:2 source: the even chroma line serves both rows (yuv2rgb.c:133-136)
        sws_unscaled_yuv2rgb24_kernel<<<dim3(((p.dstW >> 1) + 255) / 256, p.dstH >> 1, nframes), 256, 0, st>>>(p, a);
        if (check_launch("sws_scale:unscaled")) return -1;
        break;
    }
    case R_RGB48:
        sws_rgb48_kernel<<<dim3((((p.dstW + 1) >> 1) + 127) / 128, p.dstH, nframes), 128, 0, st>>>(p, fused_args(src, srcStride, srcFrame, dst[0], dstStride[0], dstFrame[0]));
        return check_launch("sws_scale:rgb48");
    case R_FUSED:
        if (run_fused(c, src, srcStride, srcFrame, dst, dstStride, dstFrame, nframes, st)) return -1;
        break;
    case R_SCALE:
        if (run_scale(c, src, srcStride, srcFrame, dst, dstStride, dstFrame, nframes, st)) return -1;
        break;
    }
    if (!expand) return 0;
    const int cols = packed_cols(c, dstStride_[0], srcStride_);
    sws_expand_rgb32_kernel<<<dim3((cols + 255) / 256, p.dstH, nframes), 256, 0, st>>>(c->d_rgb, pitch32, frame32, dst_[0], dstStride_[0], dstFrame_[0], cols, D->r, D->g, D->b, D->a);
    return check_launch("sws_scale:rgb32");
}

bool sws_slot_view(const void *ctx, SwsSlotView &v)
{
    const SwsCudaContext *c = (const SwsCudaContext *)ctx;
    if (!c) return false;
    const PixFmt *D = c->D;
    v.rangeConv = c->rangeConv; v.srcBits = c->srcFmt->bits;
    v.k = c->k; v.flags = c->g.flags; v.planar = is_planar(D); v.dstBits = D->bits; v.dstBE = D->be; v.dstNV = D->fam == FAM_NV ? 1 + (D->fmt == PIX_NV21) : 0;
    if (D->rgb16 || D->rgb48 || c->dstFmt->fam == FAM_GRAY || c->srcFmt->fam == FAM_GRAY) return false; // (the per-line slots do not cover the 15 / 16 / 12 / 48-bpp output stages: the hook leaves the C slots)
    v.target = D->slot;
    return true;
}

}  // namespace avb

using namespace avb;

extern "C" {

SwsContextCUDA *sws_getContext_cuda(int srcW, int srcH, int srcFormat, int dstW, int dstH, int dstFormat, int flags,
                                    void *srcFilter, void *dstFilter, const double *param)
{
    avb::enter();
    return (SwsContextCUDA *)make_context(srcW, srcH, srcFormat, dstW, dstH, dstFormat, flags, param, true, srcFilter, dstFilter);
}

void sws_freeContext_cuda(SwsContextCUDA *ctx) { avb::enter(); sws_slots_forget(ctx); destroy((SwsCudaContext *)ctx); }

// sws_setColorspaceDetails (libswscale/utils.c:807-835): new yuv -> rgb constants (ff_yuv2rgb_c_init_tables, yuv2rgb.c:671-863) for a
// packed rgb destination; -1 for yuv destinations like the reference, and -1 (nothing changed) for what is not taken over.
int sws_setColorspaceDetails_cuda(SwsContextCUDA *ctx, const int inv_table[4], int srcRange, const int table[4], int dstRange,
                                  int brightness, int contrast, int saturation)
{
    avb::enter();
    SwsCudaContext *c = (SwsCudaContext *)ctx;
    (void)table; (void)dstRange;                  // only read by the yuv -> yuv range conversion (not taken over) and rgb sources' fixed readers
    if (!c || !inv_table) { set_error_msg("sws_setColorspaceDetails_cuda", "NULL argument"); return -1; }
    if (is_planar(c->D) || c->D->pk422) return -1;         // isYUV(dstFormat): the reference returns -1 as well (utils.c:821-822)
    if (!ROUTES[c->route].tables) return 0;       // rgb -> rgb copies / swaps never look at the tables
    RgbConstants k;
    rgb_constants(k, inv_table, srcRange != 0, brightness, contrast, saturation);
    if (k.cy <= 0) { set_error_msg("sws_setColorspaceDetails_cuda", "contrast must be positive"); return -1; }
    // the reference indexes a 1024-entry table with Y + offset(U, V): the settings must keep every index inside it
    const int lo[3] = { k.ar + (int)std::min<int64_t>(0, (255LL * k.crv) >> 16), k.agu + k.agv + (int)std::min<int64_t>(0, (255LL * k.cgu) >> 16) + (int)std::min<int64_t>(0, (255LL * k.cgv) >> 16),
                        k.ab + (int)std::min<int64_t>(0, (255LL * k.cbu) >> 16) };
    const int hi[3] = { k.ar + (int)std::max<int64_t>(0, (255LL * k.crv) >> 16), k.agu + k.agv + (int)std::max<int64_t>(0, (255LL * k.cgu) >> 16) + (int)std::max<int64_t>(0, (255LL * k.cgv) >> 16),
                        k.ab + (int)std::max<int64_t>(0, (255LL * k.cbu) >> 16) };
    for (int ch = 0; ch < 3; ch++)
        if (lo[ch] < 0 || hi[ch] + 255 > 1023) { set_error_msg("sws_setColorspaceDetails_cuda", "these settings index outside the reference's colour table"); return -1; }
    c->k = k; c->dev.k = k; c->srcRange = srcRange != 0;
    return 0;
}

int sws_scale_frames_cuda(SwsContextCUDA *ctx, const uint8_t *const src[3], const int srcStride[3], const size_t srcFrameStride[3],
                          uint8_t *const dst[3], const int dstStride[3], const size_t dstFrameStride[3], int nframes, void *stream)
{
    avb::enter();
    SwsCudaContext *c = (SwsCudaContext *)ctx;
    if (!c) { set_error_msg("sws_scale_frames_cuda", "NULL context"); return -1; }
    static const size_t zero3[3] = { 0, 0, 0 };
    const size_t *srcFrame = srcFrameStride ? srcFrameStride : zero3, *dstFrame = dstFrameStride ? dstFrameStride : zero3;
    const uint8_t *s3[3]; int ss3[3]; size_t sf3[3];
    if (c->srcFmt->fam == FAM_GRAY && src && src[0] && srcStride && (!src[1] || !src[2])) {     // one plane: the luma plane stands in for the two nobody reads
        for (int p = 0; p < 3; p++) { s3[p] = src[0]; ss3[p] = srcStride[0]; sf3[p] = srcFrame[0]; }
        src = s3; srcStride = ss3; srcFrame = sf3;
    }
    uint8_t *d3[3]; int ds3[3]; size_t df3[3];
    if (c->dstFmt->fam == FAM_GRAY && dst && dst[0] && dstStride) {       // chroma to scratch (every frame of the batch into the same two planes: nobody reads them)
        d3[0] = dst[0]; d3[1] = c->d_gray[0]; d3[2] = c->d_gray[1];
        ds3[0] = dstStride[0]; ds3[1] = ds3[2] = c->grayPitch;
        df3[0] = dstFrame[0]; df3[1] = df3[2] = 0;
        dst = d3; dstStride = ds3; dstFrame = df3;
    } else if (c->S->fam == FAM_PAL8 && src && !src[1]) {
        set_error_msg("sws_scale_frames_cuda", "a pal8 batch needs its palettes in plane 1 (device pointer, 1024 bytes per frame)"); return -1;
    }
    const bool pk = is_packed_src(c->S), nv = c->S->fam == FAM_NV;
    if (!src || !dst || !src[0] || (!pk && (!src[1] || (!nv && !src[2]))) || !dst[0] || (is_planar(c->D) && (!dst[1] || (c->D->fam != FAM_NV && !dst[2])))) {
        set_error_msg("sws_scale_frames_cuda", "bad image pointers"); return -1;
    }
    if (run_frames(c, src, srcStride, srcFrame, dst, dstStride, dstFrame, nframes, (cudaStream_t)stream)) return -1;
    return c->g.dstH * nframes;
}

static int scale_host(SwsCudaContext *c, const uint8_t *const srcSlice[], const int srcStride[], int srcSliceY, int srcSliceH,
                      uint8_t *const dst[], const int dstStride[]);

// Bottom-up pictures (negative strides, e.g. after a vertical flip that only negates linesize; the reference handles them like any
// other stride, swscale_unscaled.c:1212-1340): the planes with a negative stride are copied row by row into top-down host buffers of the
// same pitch, the call below runs on those, and destination planes are copied back the same way (pre-filled with the caller's bytes so
// that what a converter leaves untouched stays untouched).  Rows are copied with a few bytes past the nominal width -- the bytes the
// top-down path may look at or write (odd widths, pair rounding) -- never more than the pitch.
static int sws_scale_cuda_flipped(SwsCudaContext *c, const uint8_t *const srcSlice[], const int srcStride[], int srcSliceH, uint8_t *const dst[], const int dstStride[])
{
    const PlaneGeom S = src_planes(c), D = dst_planes(c);
    std::vector<uint8_t> sbuf[3], dbuf[3];
    const uint8_t *s2[4] = { nullptr, nullptr, nullptr, nullptr };
    uint8_t *d2[4] = { nullptr, nullptr, nullptr, nullptr };
    int ss[4] = { 0, 0, 0, 0 }, ds[4] = { 0, 0, 0, 0 };
    size_t drow[3] = { 0, 0, 0 };
    if (c->S->fam == FAM_PAL8) { s2[1] = srcSlice[1]; ss[1] = srcStride[1]; }       // (pal8: the palette travels as it is)
    for (int p = 0; p < S.n; p++) {
        s2[p] = srcSlice[p]; ss[p] = srcStride[p];
        if (srcStride[p] >= 0) continue;
        const size_t pitch = (size_t)(-(ptrdiff_t)srcStride[p]), row = std::min(pitch, S.row[p] + 16);
        sbuf[p].assign(pitch * S.rows[p] + 16, 0);
        for (int y = 0; y < S.rows[p]; y++) memcpy(sbuf[p].data() + y * pitch, srcSlice[p] + (ptrdiff_t)y * srcStride[p], row);
        s2[p] = sbuf[p].data(); ss[p] = (int)pitch;
    }
    for (int p = 0; p < D.n; p++) {
        d2[p] = dst[p]; ds[p] = dstStride[p];
        if (dstStride[p] >= 0) continue;
        const size_t pitch = (size_t)(-(ptrdiff_t)dstStride[p]);
        drow[p] = std::min(pitch, D.row[p] + 16);
        dbuf[p].assign(pitch * D.rows[p] + 16, 0);
        for (int y = 0; y < D.rows[p]; y++) memcpy(dbuf[p].data() + y * pitch, dst[p] + (ptrdiff_t)y * dstStride[p], drow[p]);
        d2[p] = dbuf[p].data(); ds[p] = (int)pitch;
    }
    const int r = scale_host(c, s2, ss, 0, srcSliceH, d2, ds);
    if (r <= 0) return r;
    for (int p = 0; p < D.n; p++)
        if (dstStride[p] < 0)
            for (int y = 0; y < D.rows[p]; y++) memcpy(dst[p] + (ptrdiff_t)y * dstStride[p], dbuf[p].data() + (size_t)y * ds[p], drow[p]);
    return r;
}

// Slices (libswscale/swscale_unscaled.c:1212-1340 sws_scale, libswscale/swscale.c:323-721 swscale): srcSlice[] points at source row
// srcSliceY (chroma row srcSliceY >> chrSrcVSubSample), dst[] at the top of the destination picture, and each call returns the output
// rows it completed.  The rows received so far are kept in the context; a call runs the frame pipeline over them and hands back the rows
// the reference would have finished with the same slices: for its scaler loop all dstY whose last luma line (of the chroma-aligned row
// group, lastLumSrcY2) and last chroma line lie inside the rows received ("enough_lines", swscale.c:483-485), for its unscaled converters
// the rows of the slice itself.  Top-down, contiguous slices only (srcSliceY == 0 restarts a picture); a slice costs a whole-frame pass.
static int sws_scale_cuda_sliced(SwsCudaContext *c, const uint8_t *const srcSlice[], const int srcStride[], int srcSliceY, int srcSliceH,
                                 uint8_t *const dst[], const int dstStride[])
{
    const SwsGeometry &g = c->g;
    const PlaneGeom S = src_planes(c), D = dst_planes(c);
    const RouteFacts &rf = ROUTES[c->route];
    if (srcSliceY < 0 || srcSliceH < 0 || srcSliceY + srcSliceH > g.srcH) { set_error_msg("sws_scale_cuda", "slice outside the picture"); return 0; }
    for (int p = 0; p < S.n; p++) if (srcStride[p] < 0) { set_error_msg("sws_scale_cuda", "slices of bottom-up pictures are not taken over"); return 0; }
    for (int p = 0; p < D.n; p++) if (dstStride[p] < 0) { set_error_msg("sws_scale_cuda", "slices of bottom-up pictures are not taken over"); return 0; }
    if (srcSliceY == 0) { c->sliceNextY = 0; c->sliceDstY = 0; }
    else if (srcSliceY != c->sliceNextY) {
        // (the reference also takes bottom-up slice orders, and answers "Slices start in the middle!" to a first slice that touches neither end)
        set_error_msg("sws_scale_cuda", "slices are taken over top-down and contiguous only"); return 0;
    }
    const int end = srcSliceY + srcSliceH;
    {
        // a slice boundary inside a source chroma row makes the reference's scaler loop address rows before the slice (it has no check for it);
        // the unscaled converters work on whole chroma row groups of either side
        const int sub = rf.rowMapped ? std::max({ g.chrSrcVSub, g.chrDstVSub, rf.chrAlign }) : g.chrSrcVSub;
        const int m = (1 << sub) - 1;
        if ((srcSliceY & m) || ((srcSliceH & m) && end != g.srcH)) { set_error_msg("sws_scale_cuda", "slice not aligned to the chroma rows"); return 0; }
    }
    // keep the rows
    const int cY0 = srcSliceY >> g.chrSrcVSub, cY1 = -((-end) >> g.chrSrcVSub);
    for (int p = 0; p < S.n; p++) {
        const size_t pitch = (size_t)srcStride[p];
        if (c->sliceSrc[p].size() != pitch * S.rows[p] + 16 || c->slicePitch[p] != srcStride[p]) {
            if (srcSliceY != 0) { set_error_msg("sws_scale_cuda", "the source pitch changed between slices"); return 0; }
            c->sliceSrc[p].assign(pitch * S.rows[p] + 16, 0);
            c->slicePitch[p] = srcStride[p];
        }
        const int y0 = p ? cY0 : srcSliceY, y1 = p ? (cY1 < S.rows[p] ? cY1 : S.rows[p]) : end;
        const size_t row = pitch < S.row[p] + 16 ? pitch : S.row[p] + 16;
        for (int y = y0; y < y1; y++) memcpy(c->sliceSrc[p].data() + (size_t)y * pitch, srcSlice[p] + (size_t)(y - y0) * pitch, row);
    }
    // the output rows this slice completes
    int dstY0, dstY1;
    if (rf.rowMapped) { dstY0 = srcSliceY; dstY1 = end; }
    else {
        const int cdv = g.chrDstVSub, vL = c->vLum.size, vC = c->vChr.size;
        dstY0 = c->sliceDstY;
        for (dstY1 = dstY0; dstY1 < g.dstH; dstY1++) {
            const int grp = dstY1 | ((1 << cdv) - 1), last = grp < g.dstH - 1 ? grp : g.dstH - 1;
            const int fl = c->vLum.pos[last] > 1 - vL ? c->vLum.pos[last] : 1 - vL, fc = c->vChr.pos[dstY1 >> cdv] > 1 - vC ? c->vChr.pos[dstY1 >> cdv] : 1 - vC;
            const int ll = (g.srcH < fl + vL ? g.srcH : fl + vL) - 1, lc = (g.chrSrcH < fc + vC ? g.chrSrcH : fc + vC) - 1;
            if (!(ll < end && lc < cY1)) break;
        }
    }
    c->sliceNextY = end == g.srcH ? 0 : end;
    c->sliceDstY = end == g.srcH ? 0 : dstY1;
    const int ret = rf.rowMapped ? srcSliceH : dstY1 - dstY0;
    if (dstY1 <= dstY0) return ret;
    // the frame pipeline over the rows so far, into a copy of the caller's picture; the finished rows go back
    std::vector<uint8_t> dbuf[3];
    const uint8_t *s2[4] = { nullptr, nullptr, nullptr, nullptr };
    uint8_t *d2[4] = { nullptr, nullptr, nullptr, nullptr };
    int ss[4] = { 0, 0, 0, 0 }, ds[4] = { 0, 0, 0, 0 };
    size_t drow[3] = { 0, 0, 0 };
    for (int p = 0; p < S.n; p++) { s2[p] = c->sliceSrc[p].data(); ss[p] = srcStride[p]; }
    if (c->S->fam == FAM_PAL8) { s2[1] = srcSlice[1]; ss[1] = srcStride[1]; }         // (pal8: this slice's palette, like sws_scale() rebuilds its tables per call)
    for (int p = 0; p < D.n; p++) {
        const size_t pitch = (size_t)dstStride[p];
        drow[p] = pitch < D.row[p] + 16 ? pitch : D.row[p] + 16;
        dbuf[p].assign(pitch * D.rows[p] + 16, 0);
        for (int y = 0; y < D.rows[p]; y++) memcpy(dbuf[p].data() + (size_t)y * pitch, dst[p] + (size_t)y * pitch, drow[p]);
        d2[p] = dbuf[p].data(); ds[p] = dstStride[p];
    }
    if (scale_host(c, s2, ss, 0, g.srcH, d2, ds) <= 0) return 0;
    c->sliceNextY = end == g.srcH ? 0 : end;          // (the whole-frame call above restarted the slice state)
    c->sliceDstY = end == g.srcH ? 0 : dstY1;
    const int s = 1 << g.chrDstVSub;
    for (int p = 0; p < D.n; p++) {
        const int y0 = p ? (dstY0 + s - 1) >> g.chrDstVSub : dstY0;
        int y1 = p ? (dstY1 + s - 1) >> g.chrDstVSub : dstY1;
        if (y1 > D.rows[p]) y1 = D.rows[p];
        for (int y = y0; y < y1; y++) memcpy(dst[p] + (size_t)y * ds[p], dbuf[p].data() + (size_t)y * ds[p], drow[p]);
    }
    return ret;
}

// Host-pointer drop-in for sws_scale() (libswscale/swscale_unscaled.c:1212-1340): whole frames, or top-down slices (above).
// Returns the number of output lines like the reference, 0 on bad arguments.
int sws_scale_cuda(SwsContextCUDA *ctx, const uint8_t *const srcSlice[], const int srcStride[], int srcSliceY, int srcSliceH,
                   uint8_t *const dst[], const int dstStride[])
{
    avb::enter();
    SwsCudaContext *c = (SwsCudaContext *)ctx;
    if (!c || srcSliceH == 0) return 0;
    const uint8_t *s4[4]; int ss4[4];
    if (c->srcFmt->fam == FAM_GRAY && srcSlice && srcSlice[0] && srcStride && (!srcSlice[1] || !srcSlice[2] || srcStride[1] != srcStride[0] || srcStride[2] != srcStride[0])) {
        // a gray8 picture has one plane (data[1] of an AVFrame is its pseudo-palette): the luma plane stands in for the two planes nobody reads
        for (int p = 0; p < 3; p++) { s4[p] = srcSlice[0]; ss4[p] = srcStride[0]; }
        s4[3] = nullptr; ss4[3] = 0;
        srcSlice = s4; srcStride = ss4;
    }
    uint8_t *d4[4]; int ds4[4];
    if (c->dstFmt->fam == FAM_GRAY && dst && dst[0] && dstStride) {        // (a gray8 caller's dst[] has one plane)
        if (srcSliceY != 0 || srcSliceH != c->g.srcH) {
            // the rows a slice completes follow the destination's chroma geometry; a gray8 destination has none in the reference (chrDstVSubSample 0,
            // its own vertical chroma filter) while this context carries the planar stand-in's: whole frames only
            set_error_msg("sws_scale_cuda", "slices into a gray8 destination are not taken over (whole frames are)"); return 0;
        }
        // the chroma planes of the planar conversion go to host scratch of the context (they are computed and dropped); bottom-up: the scratch
        // planes are addressed from their last row like the caller's plane
        const size_t bytes = (size_t)c->grayPitch * (c->g.chrDstH + 2);
        const bool up = dstStride[0] < 0;
        for (int k = 0; k < 2; k++) {
            if (c->h_gray[k].size() < bytes) c->h_gray[k].resize(bytes);
            d4[1 + k] = c->h_gray[k].data() + (up ? (size_t)c->grayPitch * (c->g.chrDstH - 1) : 0);
            ds4[1 + k] = up ? -c->grayPitch : c->grayPitch;
        }
        d4[0] = dst[0]; ds4[0] = dstStride[0]; d4[3] = nullptr; ds4[3] = 0;
        dst = d4; dstStride = ds4;
    }
    return scale_host(c, srcSlice, srcStride, srcSliceY, srcSliceH, dst, dstStride);
}

// sws_scale_cuda on the planes as given
static int scale_host(SwsCudaContext *c, const uint8_t *const srcSlice[], const int srcStride[], int srcSliceY, int srcSliceH,
                      uint8_t *const dst[], const int dstStride[])
{
    const bool rgb = !is_planar(c->D);
    const bool nv = c->S->fam == FAM_NV, pk = is_packed_src(c->S), dstNV = c->D->fam == FAM_NV;
    if (!srcSlice || !dst || !srcSlice[0] || !srcStride[0] || (!pk && (!srcSlice[1] || !srcStride[1] || (!nv && (!srcSlice[2] || !srcStride[2])))) ||
        !dst[0] || !dstStride[0] || (!rgb && (!dst[1] || !dstStride[1] || (!dstNV && (!dst[2] || !dstStride[2]))))) {
        set_error_msg("sws_scale_cuda", "bad image pointers"); return 0;
    }
    if (c->S->fam == FAM_PAL8 && !srcSlice[1]) { set_error_msg("sws_scale_cuda", "a pal8 picture needs its palette in plane 1"); return 0; }
    if (srcSliceY != 0 || srcSliceH != c->g.srcH) return sws_scale_cuda_sliced(c, srcSlice, srcStride, srcSliceY, srcSliceH, dst, dstStride);
    c->sliceNextY = 0; c->sliceDstY = 0;
    if (srcStride[0] < 0 || (!pk && (srcStride[1] < 0 || (!nv && srcStride[2] < 0))) || dstStride[0] < 0 ||
        (!rgb && (dstStride[1] < 0 || (!dstNV && dstStride[2] < 0))))
        return sws_scale_cuda_flipped(c, srcSlice, srcStride, srcSliceH, dst, dstStride);
    // the context's own three streams: like the reference's SwsContext a context serves one thread at a time (swscale.c:393-398), and
    // contexts of different threads run concurrently -- eight streams keep both PCIe directions busy where one leaves bubbles between
    // the frames (the host-pointer call must return a finished picture)
    if (!c->streams_ok) {
        for (int i = 0; i < 3; i++)
            if (cudaStreamCreateWithFlags(&c->streams[i], cudaStreamNonBlocking) != cudaSuccess) { set_error("sws_scale_cuda:streams", cudaGetLastError()); return 0; }
        c->streams_ok = true;
    }
    cudaStream_t *st = c->streams;
    cudaStream_t s = st[0];
    const SwsGeometry &g = c->g;
    // device staging: tight, aligned pitches (a packed source keeps the caller's pitch: the chroma readers look one pixel past an odd
    // width, into the padding or the next row; a packed destination gets room for the pixel past an odd width)
    const PlaneGeom SP = src_planes(c), DP = dst_planes(c);
    const int odd = g.dstW & 1;
    int sP[3], dP[3];
    size_t sOff[4] = { 0 }, dOff[4] = { 0 };
    for (int p = 0; p < 3; p++) {
        sP[p] = pk && !p ? srcStride[0] : (int)((SP.row[p] + 15) & ~(size_t)15);
        dP[p] = (int)((DP.row[p] + (rgb && odd ? c->D->bpp : 0) + 15) & ~(size_t)15);
        sOff[p + 1] = sOff[p] + (p < SP.n ? (size_t)sP[p] * SP.rows[p] : 0);
        dOff[p + 1] = dOff[p] + (p < DP.n ? (size_t)dP[p] * DP.rows[p] : 0);
    }
    if (grow(c->d_src, c->src_bytes, sOff[3], s, "sws_scale_cuda") || grow(c->d_dst, c->dst_bytes, dOff[3], s, "sws_scale_cuda")) return 0;
    const uint8_t *ds[3] = { c->d_src, c->S->fam == FAM_PAL8 ? c->d_pal : c->d_src + sOff[1], c->d_src + sOff[2] };     // (pal8: plane 1 is the palette)
    uint8_t *dd[3] = { c->d_dst, c->d_dst + dOff[1], c->d_dst + dOff[2] };
    // Same-size rgb (the dp4a fused kernel): the frame goes through in three bands of rows (whole tiles of four row pairs), one per
    // stream, so the upload of band k + 1, the kernel of band k and the download of band k - 1 overlap -- the call is PCIe bound and
    // PCIe is full duplex.
    // A band re-uploads the few chroma lines it shares with its neighbours (identical bytes), so bands need no cross-stream order.
    if (c->route == R_FUSED && c->fast_ok && !nv && c->D->fam == FAM_RGB24 && !odd && g.dstH >= 64 && !((uintptr_t)c->dev.vChrF & 15)) {
        const int pairs = g.dstH / 2, per = ((pairs + 2) / 3 + 3) & ~3;        // row pairs per band
        int k = 0;
        for (int rp0 = 0; rp0 < pairs; rp0 += per, k = (k + 1) % 3) {
            const int rp1 = rp0 + per < pairs ? rp0 + per : pairs, y0 = 2 * rp0, y1 = 2 * rp1;
            cudaStream_t sb = st[k];
            int clo = c->vChr.pos[y0] > -3 ? c->vChr.pos[y0] : -3, chi = (c->vChr.pos[y1 - 1] > -3 ? c->vChr.pos[y1 - 1] : -3) + 4;
            clo = clo < 0 ? 0 : clo; chi = chi > g.chrSrcH - 1 ? g.chrSrcH - 1 : chi;
            if (cudaMemcpy2DAsync((void *)(ds[0] + (size_t)y0 * sP[0]), sP[0], srcSlice[0] + (size_t)y0 * srcStride[0], srcStride[0], g.srcW, y1 - y0, cudaMemcpyHostToDevice, sb) != cudaSuccess ||
                cudaMemcpy2DAsync((void *)(ds[1] + (size_t)clo * sP[1]), sP[1], srcSlice[1] + (size_t)clo * srcStride[1], srcStride[1], g.chrSrcW, chi - clo + 1, cudaMemcpyHostToDevice, sb) != cudaSuccess ||
                cudaMemcpy2DAsync((void *)(ds[2] + (size_t)clo * sP[2]), sP[2], srcSlice[2] + (size_t)clo * srcStride[2], srcStride[2], g.chrSrcW, chi - clo + 1, cudaMemcpyHostToDevice, sb) != cudaSuccess) {
                set_error("sws_scale_cuda:h2d", cudaGetLastError()); return 0;
            }
            static const size_t zero3[3] = { 0, 0, 0 };
            FusedArgs a = fused_args(ds, sP, zero3, dd[0], dP[0], 0);
            a.rp0 = rp0; a.rp1 = rp1;
            if (launch_fused_fast(c, a, 1, sb)) return 0;
            if (cudaMemcpy2DAsync(dst[0] + (size_t)y0 * dstStride[0], dstStride[0], dd[0] + (size_t)y0 * dP[0], dP[0], (size_t)g.dstW * 3, y1 - y0, cudaMemcpyDeviceToHost, sb) != cudaSuccess) {
                set_error("sws_scale_cuda:d2h", cudaGetLastError()); return 0;
            }
        }
        for (int q = 0; q < 3; q++) if (cudaStreamSynchronize(st[q]) != cudaSuccess) { set_error("sws_scale_cuda:sync", cudaGetLastError()); return 0; }
        return g.dstH;
    }
    // planar -> packed 4:2:2 converters: the rounded-up last pair reads the samples just past the width (to422_pairs)
    int upX = 0, upCX = 0;
    if (c->route == R_422_FROM_422P || c->route == R_422_FROM_420P) {
        const int np = to422_pairs(g.srcW, dstStride[0], srcStride);
        upX = std::max(0, 2 * np - g.srcW); upCX = std::max(0, np - g.chrSrcW);
    }
    if (pk) {
        const int bpp = c->S->bpp;
        size_t rowB = (size_t)g.srcW * bpp;
        if ((g.srcW & 1) && rowB + bpp <= (size_t)srcStride[0]) rowB += bpp;       // the pixel the readers look at past an odd width
        if (cudaMemcpyAsync((void *)ds[0], srcSlice[0], (size_t)(g.srcH - 1) * srcStride[0] + rowB, cudaMemcpyHostToDevice, s) != cudaSuccess ||
            (c->S->fam == FAM_PAL8 && cudaMemcpyAsync(c->d_pal, srcSlice[1], 1024, cudaMemcpyHostToDevice, s) != cudaSuccess)) {
            set_error("sws_scale_cuda:h2d", cudaGetLastError()); return 0;
        }
    } else {
        const size_t sS = c->srcFmt->bits > 8 ? 2 : 1;
        for (int p = 0; p < SP.n; p++)
            if (cudaMemcpy2DAsync((void *)ds[p], sP[p], srcSlice[p], srcStride[p], SP.row[p] + (p ? upCX : upX) * sS, SP.rows[p], cudaMemcpyHostToDevice, s) != cudaSuccess) {
                set_error("sws_scale_cuda:h2d", cudaGetLastError()); return 0;
            }
    }
    static const size_t zero3[3] = { 0, 0, 0 };
    if (run_frames(c, ds, sP, zero3, dd, dP, zero3, 1, s)) return 0;
    cudaError_t e;
    if (rgb) {
        e = cudaMemcpy2DAsync(dst[0], dstStride[0], dd[0], dP[0], (size_t)packed_cols(c, dstStride[0], srcStride) * c->D->bpp, g.dstH, cudaMemcpyDeviceToHost, s);
    } else {
        int w, cw, ch;
        planar_extent(c, w, cw, ch);
        const size_t sB = c->D->bits > 8 ? 2 : 1;
        e = cudaMemcpy2DAsync(dst[0], dstStride[0], dd[0], dP[0], (size_t)w * sB, g.dstH, cudaMemcpyDeviceToHost, s);
        for (int p = 1; p < DP.n && e == cudaSuccess && cw && ch; p++)
            e = cudaMemcpy2DAsync(dst[p], dstStride[p], dd[p], dP[p], (size_t)cw * sB * (dstNV ? 2 : 1), ch, cudaMemcpyDeviceToHost, s);
    }
    if (e == cudaSuccess) e = cudaStreamSynchronize(s);
    if (e != cudaSuccess) { set_error("sws_scale_cuda:d2h", e); return 0; }
    return g.dstH;
}

int sws_is_fused_cuda(SwsContextCUDA *ctx) { avb::enter(); return ctx ? ((SwsCudaContext *)ctx)->route == R_FUSED : 0; }

// Host-only introspection used by the CPU test-suite to pin the set-up stage against the reference
// (no device is touched): filter bank `which` (0 hLum, 1 hChr, 2 vLum, 3 vChr) of the context that
// sws_getContext_cuda() would build.  Returns the tap count, <0 on error.
int sws_debug_filter2_cuda(int which, int srcW, int srcH, int dstW, int dstH, int dstFormat, int flags, const void *srcFilter, const void *dstFilter,
                           int16_t *filter, int32_t *pos, int cap, int *n_out);
int sws_debug_filter_cuda(int which, int srcW, int srcH, int dstW, int dstH, int dstFormat, int flags, int16_t *filter,
                          int32_t *pos, int cap, int *n_out)
{
    avb::enter();
    return sws_debug_filter2_cuda(which, srcW, srcH, dstW, dstH, dstFormat, flags, nullptr, nullptr, filter, pos, cap, n_out);
}
// the same with the caller's SwsFilter pair (libswscale/swscale.h:112-117 layout)
int sws_debug_filter2_cuda(int which, int srcW, int srcH, int dstW, int dstH, int dstFormat, int flags, const void *srcFilter, const void *dstFilter,
                           int16_t *filter, int32_t *pos, int cap, int *n_out)
{
    avb::enter();
    SwsCudaContext *c = make_context(srcW, srcH, PIX_YUV420P, dstW, dstH, dstFormat, flags, nullptr, false, srcFilter, dstFilter);
    if (!c) return -1;
    const FilterBank &b = which == 0 ? c->hLum : which == 1 ? c->hChr : which == 2 ? c->vLum : c->vChr;
    int fs = b.size;
    *n_out = b.n;
    if (b.n > cap || (int)b.coef.size() > cap) fs = -2;
    else { memcpy(filter, b.coef.data(), b.coef.size() * 2); memcpy(pos, b.pos.data(), b.pos.size() * 4); }
    delete c;
    return fs;
}
// What sws_getContext_cuda() decides for a request, without touching a device (CPU tests of the format / refusal rules):
// returns 1 and fills out[] when the request is taken over, 0 (with the error string set) when it is refused.
//   out[0] path: 1 plane copy (planarCopyWrapper / nv12ToPlanarWrapper), 2 unscaled table converter, 3 fused same-size kernel,
//          4 general scaler (tile kernel or two passes) and the 48-bit rgb kernel, 5 the unscaled converters for packed sources, rgb pairs,
//          gray8 and pal8 to rgb, 6 planar -> packed 4:2:2 converter, 7 yuv420p -> nv12 / nv21 interleave
//   out[1..4] chrSrcW, chrSrcH, chrDstW, chrDstH   out[5] source pre-pass: 0 none, 1 nv split, 2 packed reader
//   out[6] destination sample bits (planar) or bytes per pixel (packed)   out[7] full-range source
int sws_debug_plan_cuda(int srcW, int srcH, int srcFormat, int dstW, int dstH, int dstFormat, int flags, int32_t out[8])
{
    avb::enter();
    SwsCudaContext *c = make_context(srcW, srcH, srcFormat, dstW, dstH, dstFormat, flags, nullptr, false);
    if (!c) return 0;
    out[0] = ROUTES[c->route].plan;
    out[1] = c->g.chrSrcW; out[2] = c->g.chrSrcH; out[3] = c->g.chrDstW; out[4] = c->g.chrDstH;
    out[5] = is_packed_src(c->S) ? 2 : c->S->fam == FAM_NV ? 1 : 0;
    out[6] = is_planar(c->D) ? c->D->bits : c->D->bpp;
    out[7] = c->srcRange;
    delete c;
    return 1;
}
// The SwsSlotView (sws_filter.h) sws_getContext_cuda() would hand to the per-line slots, as 26 int32, computed on the host only:
// 19 colour constants, flags, planar, dstBits, dstBE, packed target, dstNV, range conversion.  Returns the count, 0 when the request is refused.
int sws_debug_slot_view_cuda(int srcW, int srcH, int srcFormat, int dstW, int dstH, int dstFormat, int flags, int32_t out[32])
{
    avb::enter();
    static_assert(sizeof(SwsSlotView) == 27 * sizeof(int32_t), "SwsSlotView is 27 ints");
    SwsCudaContext *c = make_context(srcW, srcH, srcFormat, dstW, dstH, dstFormat, flags, nullptr, false);
    if (!c) return 0;
    SwsSlotView v;
    sws_slot_view(c, v);
    memcpy(out, &v, sizeof(v));
    delete c;
    return 27;
}
void sws_debug_rgb_constants_cuda(int32_t out[10])
{
    avb::enter();
    static const int itu601[4] = { 104597, 132201, 25675, 53279 };
    RgbConstants k;
    rgb_constants(k, itu601, 0, 0, 1 << 16, 1 << 16);
    int v[10] = { k.cy, k.k1, k.crv, k.cgu, k.cgv, k.cbu, k.ar, k.agu, k.agv, k.ab };
    for (int i = 0; i < 10; i++) out[i] = v[i];
}

}  // extern "C"
