// libav_b200/csrc/faan_dct.cuh -- the floating-point AAN transforms of libavcodec: the two p8idct passes of ff_faanidct / _put / _add
// (libavcodec/faanidct.c:47-159) and row_fdct plus the column passes of ff_faandct / ff_faandct248 (libavcodec/faandct.c:70-215).
// Thread-local arithmetic only (also compiled by tests/hostsim/).
//
// Exactness.  The C code declares FLOAT as float but its A* / B* constants are double literals, and it is built without FMA.  So:
//   * every sum or difference of two FLOAT variables is a float operation;
//   * every product with a constant is a double expression: the float operand is widened, the constant (folded in double, e.g.
//     2 * (B6 - A2)) multiplies it in double, and the right-hand side -- one product, or two products and their sum -- is rounded to float
//     once, at the assignment;
//   * prescale[] / postscale[] are float roundings of the double products B_i * B_j (/ 8), and the products with them are float products;
//   * lrintf is round-half-to-even (__float2int_rn).
// nvcc contracts a * b + c into FFMA / DFMA under its default --fmad=true, so every operation below is spelled with a rounding
// intrinsic; none of them can be contracted.  Denormals are kept (no .FTZ), as on the CPU.
#pragma once
#include "common.cuh"
#ifdef AVB_HOSTSIM
#include <math.h>
#endif

namespace avb {

#ifdef AVB_HOSTSIM
// tests/hostsim/ compiles this file as host C++ for x86-64, where plain operators on float and double already round like the reference
inline float __fadd_rn(float a, float b) { return a + b; }
inline float __fsub_rn(float a, float b) { return a - b; }
inline float __fmul_rn(float a, float b) { return a * b; }
inline double __dadd_rn(double a, double b) { return a + b; }
inline double __dsub_rn(double a, double b) { return a - b; }
inline double __dmul_rn(double a, double b) { return a * b; }
inline float __double2float_rn(double x) { return (float)x; }
inline int __float2int_rn(float x) { return (int)lrintf(x); }
inline float __int_as_float(int x) { float f; memcpy(&f, &x, 4); return f; }
inline int __float_as_int(float f) { int x; memcpy(&x, &f, 4); return x; }
#endif

namespace faan {

__device__ __forceinline__ float fadd(float a, float b) { return __fadd_rn(a, b); }
__device__ __forceinline__ float fsub(float a, float b) { return __fsub_rn(a, b); }
// (float)((double)x * k): one product with a double constant, rounded to float at the assignment
__device__ __forceinline__ float mul1(float x, double k) { return __double2float_rn(__dmul_rn((double)x, k)); }
// (float)((double)x * kx + (double)y * ky), and with SUB (float)((double)x * kx - (double)y * ky): two products and their sum in double
template <bool SUB> __device__ __forceinline__ float mul2(float x, double kx, float y, double ky)
{
    const double p = __dmul_rn((double)x, kx), q = __dmul_rn((double)y, ky);
    return __double2float_rn(SUB ? __dsub_rn(p, q) : __dadd_rn(p, q));
}

// ---- faanidct.c ----
__host__ __device__ constexpr double IB(int k)
{
    return k == 0 ? 1.0000000000000000000000 : k == 1 ? 1.3870398453221474618216 : k == 2 ? 1.3065629648763765278566 : k == 3 ? 1.1758756024193587169745 :
           k == 4 ? 1.0000000000000000000000 : k == 5 ? 0.7856949583871021812779 : k == 6 ? 0.5411961001461969843997 : 0.2758993792829430123360;
}
constexpr double IA4 = 0.70710678118654752438, IA2 = 0.92387953251128675613;
// prescale[8 r + c] = B_r * B_c / 8 rounded to float (:39-48); r and c are constants after unrolling
__device__ __forceinline__ float prescale(int r, int c)
{
    return __double2float_rn(IB(r) * IB(c) / 8);
}

// one 8-point pass of p8idct (:56-97) on t[0..7]: a row (first pass) or a column (second pass); the outputs replace the inputs
__device__ __forceinline__ void idct_1d(float (&t)[8])
{
    const float s17 = fadd(t[1], t[7]), d17 = fsub(t[1], t[7]), s53 = fadd(t[5], t[3]), d53 = fsub(t[5], t[3]);
    const float od07 = fadd(s17, s53);
    float od25 = mul1(fsub(s17, s53), 2 * IA4);
    float od34 = mul2<true>(d17, 2 * (IB(6) - IA2), d53, 2 * IA2);
    float od16 = mul2<false>(d53, 2 * (IA2 - IB(2)), d17, 2 * IA2);
    od16 = fsub(od16, od07);
    od25 = fsub(od25, od16);
    od34 = fadd(od34, od25);
    const float s26 = fadd(t[2], t[6]);
    float d26 = fsub(t[2], t[6]);
    d26 = mul1(d26, 2 * IA4);
    d26 = fsub(d26, s26);
    const float s04 = fadd(t[0], t[4]), d04 = fsub(t[0], t[4]);
    const float os07 = fadd(s04, s26), os34 = fsub(s04, s26), os16 = fadd(d04, d26), os25 = fsub(d04, d26);
    t[0] = fadd(os07, od07); t[7] = fsub(os07, od07);
    t[1] = fadd(os16, od16); t[6] = fsub(os16, od16);
    t[2] = fadd(os25, od25); t[5] = fsub(os25, od25);
    t[3] = fsub(os34, od34); t[4] = fadd(os34, od34);
}

// temp[] of row r after the first pass: prescaled coefficients (:120-121), transformed along the row
__device__ __forceinline__ void idct_row(const int (&x)[8], int r, float (&t)[8])
{
#pragma unroll
    for (int c = 0; c < 8; c++) t[c] = __fmul_rn((float)x[c], prescale(r, c));
    idct_1d(t);
}

// ---- faandct.c ----
__host__ __device__ constexpr double FB(int k)
{
    return k == 0 ? 1.00000000000000000000 : k == 1 ? 0.72095982200694791383 : k == 2 ? 0.76536686473017954350 : k == 3 ? 0.85043009476725644878 :
           k == 4 ? 1.00000000000000000000 : k == 5 ? 1.27275858057283393842 : k == 6 ? 1.84775906502257351242 : 3.62450978541155137218;
}
constexpr double FA1 = 0.70710678118654752438, FA2 = 0.54119610014619698435, FA5 = 0.38268343236508977170, FA4 = 1.30656296487637652774;
// postscale[8 r + c] = B_r * B_c rounded to float (:56-65)
__device__ __forceinline__ float postscale(int r, int c)
{
    return __double2float_rn(FB(r) * FB(c));
}

// the AAN butterfly shared by row_fdct (:70-119) and ff_faandct's columns (:131-177), from its first sums / differences
// tmp0..tmp7; out[k] is the unscaled coefficient k
__device__ __forceinline__ void fdct_1d(float tmp0, float tmp1, float tmp2, float tmp3, float tmp4, float tmp5, float tmp6, float tmp7,
                                        float (&out)[8])
{
    const float tmp10 = fadd(tmp0, tmp3), tmp13 = fsub(tmp0, tmp3), tmp11 = fadd(tmp1, tmp2);
    float tmp12 = fsub(tmp1, tmp2);
    out[0] = fadd(tmp10, tmp11);
    out[4] = fsub(tmp10, tmp11);
    tmp12 = fadd(tmp12, tmp13);
    tmp12 = mul1(tmp12, FA1);
    out[2] = fadd(tmp13, tmp12);
    out[6] = fsub(tmp13, tmp12);
    tmp4 = fadd(tmp4, tmp5);
    tmp5 = fadd(tmp5, tmp6);
    tmp6 = fadd(tmp6, tmp7);
    const float z2 = mul2<true>(tmp4, FA2 + FA5, tmp6, FA5);
    const float z4 = mul2<false>(tmp6, FA4 - FA5, tmp4, FA5);
    tmp5 = mul1(tmp5, FA1);
    const float z11 = fadd(tmp7, tmp5), z13 = fsub(tmp7, tmp5);
    out[5] = fadd(z13, z2); out[3] = fsub(z13, z2);
    out[1] = fadd(z11, z4); out[7] = fsub(z11, z4);
}

// row_fdct on one row of int16 samples: the sums and differences are int, converted to float at the assignment (:78-85)
__device__ __forceinline__ void fdct_row(const int (&d)[8], float (&out)[8])
{
    fdct_1d((float)(d[0] + d[7]), (float)(d[1] + d[6]), (float)(d[2] + d[5]), (float)(d[3] + d[4]),
            (float)(d[3] - d[4]), (float)(d[2] - d[5]), (float)(d[1] - d[6]), (float)(d[0] - d[7]), out);
}

// lrintf(postscale[8 r + c] * v), the long the C code stores into int16 (the caller truncates)
__device__ __forceinline__ int scaled(float v, int r, int c) { return __float2int_rn(__fmul_rn(postscale(r, c), v)); }

// column c of ff_faandct (:131-177) on the row pass's output t[row]
__device__ __forceinline__ void fdct_col(const float (&t)[8], int c, int (&out)[8])
{
    float o[8];
    fdct_1d(fadd(t[0], t[7]), fadd(t[1], t[6]), fadd(t[2], t[5]), fadd(t[3], t[4]),
            fsub(t[3], t[4]), fsub(t[2], t[5]), fsub(t[1], t[6]), fsub(t[0], t[7]), o);
#pragma unroll
    for (int k = 0; k < 8; k++) out[k] = scaled(o[k], k, c);
}

// column c of ff_faandct248 (:190-215): the odd rows are scaled with postscale rows 0 / 4 / 2 / 6, as the C code does
__device__ __forceinline__ void fdct248_col(const float (&t)[8], int c, int (&out)[8])
{
#pragma unroll
    for (int half = 0; half < 2; half++) {
        const float a = half ? fsub(t[0], t[1]) : fadd(t[0], t[1]), b = half ? fsub(t[2], t[3]) : fadd(t[2], t[3]);
        const float e = half ? fsub(t[4], t[5]) : fadd(t[4], t[5]), f = half ? fsub(t[6], t[7]) : fadd(t[6], t[7]);
        const float tmp10 = fadd(a, f), tmp11 = fadd(b, e), tmp13 = fsub(a, f);
        float tmp12 = fsub(b, e);
        out[half]     = scaled(fadd(tmp10, tmp11), 0, c);
        out[4 + half] = scaled(fsub(tmp10, tmp11), 4, c);
        tmp12 = fadd(tmp12, tmp13);
        tmp12 = mul1(tmp12, FA1);
        out[2 + half] = scaled(fadd(tmp13, tmp12), 2, c);
        out[6 + half] = scaled(fsub(tmp13, tmp12), 6, c);
    }
}

}  // namespace faan
}  // namespace avb
