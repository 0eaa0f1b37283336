// libav_b200/csrc/xvid_idct.cuh -- the Xvid 8x8 IDCT (ff_xvid_idct, libavcodec/xvididct.c:40-289) as a transform policy of the 8-bit IDCT
// kernel (simple_idct_kernel, idctdsp.cu) and of the thread-per-block kernel (xvid_idct.cu).  Both work on the packed form the 8-bit kernel
// stages: a row is 4 words of two int16 each.  Threads never communicate here, so the file also compiles as host C++ (tests/hostsim/).
//
// Exactness (checked block for block against the compiled xvididct.c, tests/test_xvid_idct.py):
//   * every branch of idct_row (:58-140) equals its general 4 + 4-term formula, except `return 0`, which leaves the row as it was.  For int16
//     input that happens only in row 0 holding nothing but DC = -4 (16384 * -4 + 65536 == 0): that row stays {-4, 0, ...};
//   * idct_col_4 / idct_col_3 (:208-270) equal idct_col_8 (:162-206) under the conditions ff_xvid_idct selects them: they are shortcuts for
//     zero rows, so idct_col_8 always is exact and keeps the warp converged;
//   * both passes store into int16 (`short`), and every sum and product wraps at 32 bits like the C code's int arithmetic.  TAN3 = 0xAB0E is
//     the positive int 43790 there (not the negative 16-bit value the MMX version multiplies by).
#pragma once
#include "common.cuh"

namespace avb {

// row r's constants: TAB04 TAB17 TAB26 TAB35 TAB04 TAB35 TAB26 TAB17 and RND0..RND7 (:40-56).  `r` is a constant after unrolling, so
// every selection below folds to an immediate.
struct XvidRowConsts { unsigned c1, c2, c3, c4, c5, c6, c7, rnd; };
__device__ __forceinline__ XvidRowConsts xvid_row_consts(int r)
{
    const int t = (r & 3) == 0 ? 0 : (r == 1 || r == 7) ? 1 : (r == 2 || r == 6) ? 2 : 3;
    XvidRowConsts k;
    k.c1 = t == 0 ? 22725 : t == 1 ? 31521 : t == 2 ? 29692 : 26722;
    k.c2 = t == 0 ? 21407 : t == 1 ? 29692 : t == 2 ? 27969 : 25172;
    k.c3 = t == 0 ? 19266 : t == 1 ? 26722 : t == 2 ? 25172 : 22654;
    k.c4 = t == 0 ? 16384 : t == 1 ? 22725 : t == 2 ? 21407 : 19266;
    k.c5 = t == 0 ? 12873 : t == 1 ? 17855 : t == 2 ? 16819 : 15137;
    k.c6 = t == 0 ?  8867 : t == 1 ? 12299 : t == 2 ? 11585 : 10426;
    k.c7 = t == 0 ?  4520 : t == 1 ?  6270 : t == 2 ?  5906 :  5315;
    k.rnd = r == 0 ? 65536 : r == 1 ? 3597 : r == 2 ? 2260 : r == 3 ? 1203 : r == 4 ? 0 : r == 5 ? 120 : 512;
    return k;
}

// Row pass of row r on one packed row; result is the int16-truncated row, packed.  ROW_SHIFT is 11 as in the simple IDCT, so the same
// trick applies: with every term pre-multiplied by 32, bits [26:11] of each sum (the int16 the C code stores) are the upper half-word of
// the 32-bit wrap-around result, picked by a byte-permute.
__device__ __forceinline__ uint4 xvid_row(uint4 v, int r)
{
    const XvidRowConsts K = xvid_row_consts(r);
    const unsigned x0 = (unsigned)lo16s(v.x), x1 = (unsigned)hi16s(v.x), x2 = (unsigned)lo16s(v.y), x3 = (unsigned)hi16s(v.y);
    const unsigned x4 = (unsigned)lo16s(v.z), x5 = (unsigned)hi16s(v.z), x6 = (unsigned)lo16s(v.w), x7 = (unsigned)hi16s(v.w);
    const unsigned k = (32 * K.c4) * x0 + 32 * K.rnd;
    const unsigned b0 = k + (32 * K.c4) * x4, b1 = k - (32 * K.c4) * x4;
    const unsigned p = (32 * K.c2) * x2 + (32 * K.c6) * x6, q = (32 * K.c6) * x2 - (32 * K.c2) * x6;
    const unsigned e0 = b0 + p, e3 = b0 - p, e1 = b1 + q, e2 = b1 - q;
    const unsigned o0 = (32 * K.c1) * x1 + (32 * K.c3) * x3 + (32 * K.c5) * x5 + (32 * K.c7) * x7;
    const unsigned o1 = (32 * K.c3) * x1 - (32 * K.c7) * x3 - (32 * K.c1) * x5 - (32 * K.c5) * x7;
    const unsigned o2 = (32 * K.c5) * x1 - (32 * K.c1) * x3 + (32 * K.c7) * x5 + (32 * K.c3) * x7;
    const unsigned o3 = (32 * K.c7) * x1 - (32 * K.c5) * x3 + (32 * K.c3) * x5 - (32 * K.c1) * x7;
    uint4 o;
    o.x = __byte_perm(e0 + o0, e1 + o1, 0x7632);
    o.y = __byte_perm(e2 + o2, e3 + o3, 0x7632);
    o.z = __byte_perm(e3 - o3, e2 - o2, 0x7632);
    o.w = __byte_perm(e1 - o1, e0 - o0, 0x7632);
    // idct_row's `return 0` (:94-95): row 0 = {-4, 0, ...} is left as it was
    if (r == 0 && v.x == 0xfffcu && (v.y | v.z | v.w) == 0) o = v;
    return o;
}

// (c * x) >> 16 with the C code's int wrap-around (MULT, :145)
__device__ __forceinline__ unsigned xvid_mult(unsigned c, unsigned x) { return (unsigned)((int)(c * x) >> 16); }
// (int16_t)(v >> COL_SHIFT): bits [21:6], sign-extended
__device__ __forceinline__ int xvid_out(unsigned v) { return (int)(v << 10) >> 16; }

// idct_col_8 (:162-206) on one column of the row-transformed block: out[y] = the int16 the C code stores at row y
__device__ __forceinline__ void xvid_col(const unsigned (&x)[8], int (&out)[8])
{
    constexpr unsigned TAN1 = 0x32EC, TAN2 = 0x6A0A, TAN3 = 0xAB0E, SQRT2 = 0x5A82;
    // odd part
    const unsigned m0 = xvid_mult(TAN1, x[7]) + x[1], m1 = xvid_mult(TAN1, x[1]) - x[7];
    const unsigned m2 = xvid_mult(TAN3, x[5]) + x[3], m3 = xvid_mult(TAN3, x[3]) - x[5];
    const unsigned t7 = m0 + m2, t4 = m1 - m3, t0 = m0 - m2, t1 = m1 + m3;
    const unsigned t6 = 2 * xvid_mult(SQRT2, t0 + t1), t5 = 2 * xvid_mult(SQRT2, t0 - t1);
    // even part
    const unsigned e3 = xvid_mult(TAN2, x[6]) + x[2], e2 = xvid_mult(TAN2, x[2]) - x[6];
    const unsigned e0 = x[0] + x[4], e1 = x[0] - x[4];
    const unsigned a0 = e0 + e3, a3 = e0 - e3, a1 = e1 + e2, a2 = e1 - e2;
    out[0] = xvid_out(a0 + t7); out[7] = xvid_out(a0 - t7);
    out[3] = xvid_out(a3 + t4); out[4] = xvid_out(a3 - t4);
    out[1] = xvid_out(a1 + t6); out[6] = xvid_out(a1 - t6);
    out[2] = xvid_out(a2 + t5); out[5] = xvid_out(a2 - t5);
}

// the transform policy simple_idct_kernel takes (idctdsp.cu): row pass of row r on a packed row, column pass on the low (HI = 0) or high
// (HI = 1) half-words of eight packed row words.  MH (the simple IDCT's IMAD.HI shift variant) has no use here.
struct XvidIdct {
    template <bool MH> static __device__ __forceinline__ uint4 row(uint4 v, int r) { return xvid_row(v, r); }
    template <int HI, bool MH> static __device__ __forceinline__ void col(const uint32_t (&w)[8], int (&out)[8])
    {
        unsigned x[8];
#pragma unroll
        for (int k = 0; k < 8; k++) x[k] = (unsigned)(HI ? hi16s(w[k]) : lo16s(w[k]));
        xvid_col(x, out);
    }
};

}  // namespace avb
