// libav_b200/csrc/simple_idct8.cuh -- ff_simple_idct_8 on one thread's int16 block (libavcodec/simple_idct_template.c, BIT_DEPTH 8: W4 = 16383,
// ROW_SHIFT 11, COL_SHIFT 20, DC_SHIFT 3), shared by the quantiser metrics (me_cmp_enc.cu) and the DNxHD encoder (dnxhd_enc.cuh).  All
// arithmetic is 32-bit wrap-around like the C code's int arithmetic.  Thread-local only (also compiled by tests/hostsim/).
#pragma once
#include "common.cuh"

namespace avb {
namespace {

// the row pass in place
__device__ inline void enc_idct_rows(int16_t *b)
{
    constexpr int W1 = 22725, W2 = 21407, W3 = 19266, W4 = 16383, W5 = 12873, W6 = 8867, W7 = 4520;
    for (int r = 0; r < 8; r++) {
        int16_t *row = b + 8 * r;
        if (!(row[1] | row[2] | row[3] | row[4] | row[5] | row[6] | row[7])) {           // DC-only row: row[0] << DC_SHIFT (:94-106)
            const int16_t v = (int16_t)(((unsigned)row[0] << 3) & 0xffffu);
            for (int k = 0; k < 8; k++) row[k] = v;
            continue;
        }
        const unsigned x0 = (unsigned)(int)row[0], x1 = (unsigned)(int)row[1], x2 = (unsigned)(int)row[2], x3 = (unsigned)(int)row[3];
        const unsigned x4 = (unsigned)(int)row[4], x5 = (unsigned)(int)row[5], x6 = (unsigned)(int)row[6], x7 = (unsigned)(int)row[7];
        const unsigned base = W4 * x0 + (1u << 10);
        const unsigned e0 = base + W2 * x2 + W4 * x4 + W6 * x6, e1 = base + W6 * x2 - W4 * x4 - W2 * x6;
        const unsigned e2 = base - W6 * x2 - W4 * x4 + W2 * x6, e3 = base - W2 * x2 + W4 * x4 - W6 * x6;
        const unsigned o0 = W1 * x1 + W3 * x3 + W5 * x5 + W7 * x7, o1 = W3 * x1 - W7 * x3 - W1 * x5 - W5 * x7;
        const unsigned o2 = W5 * x1 - W1 * x3 + W7 * x5 + W3 * x7, o3 = W7 * x1 - W5 * x3 + W3 * x5 - W1 * x7;
        row[0] = (int16_t)((int)(e0 + o0) >> 11); row[7] = (int16_t)((int)(e0 - o0) >> 11);
        row[1] = (int16_t)((int)(e1 + o1) >> 11); row[6] = (int16_t)((int)(e1 - o1) >> 11);
        row[2] = (int16_t)((int)(e2 + o2) >> 11); row[5] = (int16_t)((int)(e2 - o2) >> 11);
        row[3] = (int16_t)((int)(e3 + o3) >> 11); row[4] = (int16_t)((int)(e3 - o3) >> 11);
    }
}
// the column pass of column c (c points at its first coefficient); out is not yet truncated to int16
__device__ inline void enc_idct_col(const int16_t *c, int (&out)[8])
{
    constexpr int W1 = 22725, W2 = 21407, W3 = 19266, W4 = 16383, W5 = 12873, W6 = 8867, W7 = 4520;
    const unsigned x0 = (unsigned)(int)c[0], x1 = (unsigned)(int)c[8], x2 = (unsigned)(int)c[16], x3 = (unsigned)(int)c[24];
    const unsigned x4 = (unsigned)(int)c[32], x5 = (unsigned)(int)c[40], x6 = (unsigned)(int)c[48], x7 = (unsigned)(int)c[56];
    const unsigned base = W4 * (x0 + ((1u << 19) / W4));                                  // rounding folded into the DC term (:176)
    const unsigned e0 = base + W2 * x2 + W4 * x4 + W6 * x6, e1 = base + W6 * x2 - W4 * x4 - W2 * x6;
    const unsigned e2 = base - W6 * x2 - W4 * x4 + W2 * x6, e3 = base - W2 * x2 + W4 * x4 - W6 * x6;
    const unsigned o0 = W1 * x1 + W3 * x3 + W5 * x5 + W7 * x7, o1 = W3 * x1 - W7 * x3 - W1 * x5 - W5 * x7;
    const unsigned o2 = W5 * x1 - W1 * x3 + W7 * x5 + W3 * x7, o3 = W7 * x1 - W5 * x3 + W3 * x5 - W1 * x7;
    out[0] = (int)(e0 + o0) >> 20; out[7] = (int)(e0 - o0) >> 20; out[1] = (int)(e1 + o1) >> 20; out[6] = (int)(e1 - o1) >> 20;
    out[2] = (int)(e2 + o2) >> 20; out[5] = (int)(e2 - o2) >> 20; out[3] = (int)(e3 + o3) >> 20; out[4] = (int)(e3 - o3) >> 20;
}

}  // namespace
}  // namespace avb
