// libav_b200/csrc/idct10.cuh -- the 10-bit simple IDCT's row and column passes on packed int16 pairs (simple_idct_template.c with
// BIT_DEPTH 10, :63-78), shared by the 10-bit IDCT (idct10.cu) and ProRes (prores.cu).  All arithmetic is 32-bit wrap-around like the C
// code's int arithmetic.  The row pass takes a policy: the plain transform (Simple10Rows) or ff_prores_idct's (ProresRows,
// idctRowCondDC_10(row, extra_shift = 2), simple_idct.c:222-234).  The column pass is idctSparseCol_10 for both.
#pragma once
#include "common.cuh"

namespace avb {
namespace {

constexpr unsigned K1 = 90901, K2 = 85627, K3 = 77062, K4 = 65535, K5 = 51491, K6 = 35468, K7 = 18081;      // simple_idct_template.c:63-78

// the row pass of ff_simple_idct_*_10: ROW_SHIFT 15, a DC-only row holds row[0] << DC_SHIFT (1)
struct Simple10Rows {
    static constexpr int SHIFT = 15;
    __device__ __forceinline__ static unsigned dc(unsigned x0) { return (x0 << 1) & 0xffffu; }
};
// extra_shift 2: a full row shifts by 17 but keeps the rounding constant 1 << 14; a DC-only row holds row[0] >> 1 (arithmetic, unrounded)
struct ProresRows {
    static constexpr int SHIFT = 17;
    __device__ __forceinline__ static unsigned dc(unsigned x0) { return (unsigned)((int)x0 >> 1) & 0xffffu; }
};

// even / odd halves shared by both passes (32-bit wrap-around like the C code's int arithmetic)
__device__ __forceinline__ void i10_butterfly(unsigned base, unsigned x1, unsigned x2, unsigned x3, unsigned x4, unsigned x5, unsigned x6, unsigned x7,
                                              unsigned (&s)[4], unsigned (&d)[4])
{
    const unsigned b0 = base + K4 * x4, b1 = base - K4 * x4, p = K2 * x2 + K6 * x6, q = K6 * x2 - K2 * x6;
    const unsigned e0 = b0 + p, e3 = b0 - p, e1 = b1 + q, e2 = b1 - q;
    const unsigned o0 = K1 * x1 + K3 * x3 + K5 * x5 + K7 * x7, o1 = K3 * x1 - K7 * x3 - K1 * x5 - K5 * x7;
    const unsigned o2 = K5 * x1 - K1 * x3 + K7 * x5 + K3 * x7, o3 = K7 * x1 - K5 * x3 + K3 * x5 - K1 * x7;
    s[0] = e0 + o0; s[1] = e1 + o1; s[2] = e2 + o2; s[3] = e3 + o3;
    d[0] = e0 - o0; d[1] = e1 - o1; d[2] = e2 - o2; d[3] = e3 - o3;
}
template <class P = Simple10Rows> __device__ __forceinline__ uint4 i10_row(uint4 r)
{
    const unsigned x0 = (unsigned)lo16s(r.x);
    if (((r.x & 0xffff0000u) | r.y | r.z | r.w) == 0) {                  // DC-only row: the policy's DC value in every position (:94-106)
        unsigned v = P::dc(x0); v |= v << 16;
        return make_uint4(v, v, v, v);
    }
    unsigned s[4], d[4];
    i10_butterfly(K4 * x0 + (1u << 14), (unsigned)hi16s(r.x), (unsigned)lo16s(r.y), (unsigned)hi16s(r.y), (unsigned)lo16s(r.z), (unsigned)hi16s(r.z),
                  (unsigned)lo16s(r.w), (unsigned)hi16s(r.w), s, d);
    constexpr int S = P::SHIFT;
    return make_uint4(pack16((int)s[0] >> S, (int)s[1] >> S), pack16((int)s[2] >> S, (int)s[3] >> S),
                      pack16((int)d[3] >> S, (int)d[2] >> S), pack16((int)d[1] >> S, (int)d[0] >> S));
}
template <int HI> __device__ __forceinline__ void i10_col(const uint32_t (&w)[8], int (&out)[8])
{
    unsigned x[8];
#pragma unroll
    for (int k = 0; k < 8; k++) x[k] = (unsigned)(HI ? hi16s(w[k]) : lo16s(w[k]));
    unsigned s[4], d[4];
    i10_butterfly(K4 * (x[0] + ((1u << 19) / K4)), x[1], x[2], x[3], x[4], x[5], x[6], x[7], s, d);      // rounding folded into the DC term, :176
#pragma unroll
    for (int k = 0; k < 4; k++) { out[k] = (int)s[k] >> 20; out[7 - k] = (int)d[k] >> 20; }
}
__device__ __forceinline__ int i10_clip(int v) { return min(max(v, 0), 1023); }

}  // namespace
}  // namespace avb
