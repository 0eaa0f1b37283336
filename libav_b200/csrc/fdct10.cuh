// libav_b200/csrc/fdct10.cuh -- the passes of the 10-bit accurate integer forward DCT (libavcodec/jfdctint_template.c with BIT_DEPTH 10:
// CONST_BITS 13, PASS1_BITS 1, OUT_SHIFT 2, :126-130).  Shared by fdct10.cu (ff_jpeg_fdct_islow_10 / ff_fdct248_islow_10) and the ProRes
// encoder (prores_enc.cu: prores_fdct).
#pragma once
#include "common.cuh"

namespace avb {

__device__ __forceinline__ int f10_rr(int v, int n) { return (v + (1 << (n - 1))) >> n; }
// one accurate 8-point pass; outputs 0 and 4 are scaled up by `up` bits (up < 0: rounded right shift), the rest descaled by `dn`
__device__ inline void f10_islow_1d(const int (&in)[8], int (&out)[8], int up, int dn)
{
    constexpr int K0298 = 2446, K0390 = 3196, K0541 = 4433, K0765 = 6270, K0899 = 7373, K1175 = 9633, K1501 = 12299,
                  K1847 = 15137, K1961 = 16069, K2053 = 16819, K2562 = 20995, K3072 = 25172;
    const int s0 = in[0] + in[7], d0 = in[0] - in[7], s1 = in[1] + in[6], d1 = in[1] - in[6];
    const int s2 = in[2] + in[5], d2 = in[2] - in[5], s3 = in[3] + in[4], d3 = in[3] - in[4];
    const int e0 = s0 + s3, e3 = s0 - s3, e1 = s1 + s2, e2 = s1 - s2;
    out[0] = up >= 0 ? (e0 + e1) * (1 << up) : f10_rr(e0 + e1, -up);
    out[4] = up >= 0 ? (e0 - e1) * (1 << up) : f10_rr(e0 - e1, -up);
    const int z = (e2 + e3) * K0541;
    out[2] = f10_rr(z + e3 * K0765, dn);
    out[6] = f10_rr(z - e2 * K1847, dn);
    int z1 = d3 + d0, z2 = d2 + d1, z3 = d3 + d1, z4 = d2 + d0;
    const int z5 = (z3 + z4) * K1175, t4 = d3 * K0298, t5 = d2 * K2053, t6 = d1 * K3072, t7 = d0 * K1501;
    z1 *= -K0899; z2 *= -K2562; z3 = z3 * -K1961 + z5; z4 = z4 * -K0390 + z5;
    out[7] = f10_rr(t4 + z1 + z3, dn); out[5] = f10_rr(t5 + z2 + z4, dn); out[3] = f10_rr(t6 + z2 + z3, dn); out[1] = f10_rr(t7 + z1 + z4, dn);
}
// 2-4-8 column pass: two interleaved 4-point transforms (jfdctint_template.c:342-398)
__device__ inline void f10_248_col(const int (&in)[8], int (&out)[8], int sh, int dn)
{
    constexpr int K0541 = 4433, K0765 = 6270, K1847 = 15137;
    const int a0 = in[0] + in[1], a1 = in[2] + in[3], a2 = in[4] + in[5], a3 = in[6] + in[7];
    const int b0 = in[0] - in[1], b1 = in[2] - in[3], b2 = in[4] - in[5], b3 = in[6] - in[7];
    int e0 = a0 + a3, e1 = a1 + a2, e2 = a1 - a2, e3 = a0 - a3, z;
    out[0] = f10_rr(e0 + e1, sh); out[4] = f10_rr(e0 - e1, sh);
    z = (e2 + e3) * K0541;
    out[2] = f10_rr(z + e3 * K0765, dn); out[6] = f10_rr(z - e2 * K1847, dn);
    e0 = b0 + b3; e1 = b1 + b2; e2 = b1 - b2; e3 = b0 - b3;
    out[1] = f10_rr(e0 + e1, sh); out[5] = f10_rr(e0 - e1, sh);
    z = (e2 + e3) * K0541;
    out[3] = f10_rr(z + e3 * K0765, dn); out[7] = f10_rr(z - e2 * K1847, dn);
}

}  // namespace avb
