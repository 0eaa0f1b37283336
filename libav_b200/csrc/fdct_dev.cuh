// libav_b200/csrc/fdct_dev.cuh -- one-dimensional passes of the forward DCTs of FDCTDSPContext, shared by the batched transforms (me_cmp.cu),
// the dct_* comparison metrics (me_cmp.cu) and the quantiser metrics (me_cmp_enc.cu).
//   islow_1d<UP, DN>  jpeg_fdct_islow_8 (libavcodec/jfdctint_template.c:182-338): rows <4, 9> (PASS1_BITS up, CONST_BITS - PASS1_BITS down),
//                     columns <-4, 17>
//   col_248<FAST>     the column pass of the 2-4-8 variants (jfdctint_template.c:340-398, jfdctfst.c:234-332)
//   ifast_1d          ff_fdct_ifast (libavcodec/jfdctfst.c:141-232), both passes
//   faan::*           ff_faandct / ff_faandct248 (libavcodec/faandct.c), faan_dct.cuh
// Thread-local arithmetic only (also compiled by tests/hostsim/).
#pragma once
#include "common.cuh"
#include "faan_dct.cuh"

namespace avb {

enum { K0298 = 2446, K0390 = 3196, K0541 = 4433, K0765 = 6270, K0899 = 7373, K1175 = 9633, K1501 = 12299,
       K1847 = 15137, K1961 = 16069, K2053 = 16819, K2562 = 20995, K3072 = 25172 };
__device__ __forceinline__ int rsr(int v, int n) { return (v + (1 << (n - 1))) >> n; }
__device__ __forceinline__ int fmul8(int v, int k) { return (int)(int16_t)((v * k) >> 8); }

template <int UP, int DN> __device__ __forceinline__ void islow_1d(const int (&in)[8], int (&out)[8])
{
    int s0 = in[0] + in[7], d0 = in[0] - in[7], s1 = in[1] + in[6], d1 = in[1] - in[6];
    int s2 = in[2] + in[5], d2 = in[2] - in[5], s3 = in[3] + in[4], d3 = in[3] - in[4];
    int e0 = s0 + s3, e3 = s0 - s3, e1 = s1 + s2, e2 = s1 - s2;
    out[0] = UP >= 0 ? (e0 + e1) * (1 << (UP >= 0 ? UP : 0)) : rsr(e0 + e1, UP < 0 ? -UP : 1);
    out[4] = UP >= 0 ? (e0 - e1) * (1 << (UP >= 0 ? UP : 0)) : rsr(e0 - e1, UP < 0 ? -UP : 1);
    int z = (e2 + e3) * K0541;
    out[2] = rsr(z + e3 * K0765, DN);
    out[6] = rsr(z - e2 * K1847, DN);
    int z1 = d3 + d0, z2 = d2 + d1, z3 = d3 + d1, z4 = d2 + d0, z5 = (z3 + z4) * K1175;
    int t4 = d3 * K0298, t5 = d2 * K2053, t6 = d1 * K3072, t7 = d0 * K1501;
    z1 *= -K0899; z2 *= -K2562; z3 = z3 * -K1961 + z5; z4 = z4 * -K0390 + z5;
    out[7] = rsr(t4 + z1 + z3, DN); out[5] = rsr(t5 + z2 + z4, DN); out[3] = rsr(t6 + z2 + z3, DN); out[1] = rsr(t7 + z1 + z4, DN);
}
template <bool FAST> __device__ __forceinline__ void col_248(const int (&in)[8], int (&out)[8])
{
    int a0 = in[0] + in[1], a1 = in[2] + in[3], a2 = in[4] + in[5], a3 = in[6] + in[7];
    int b0 = in[0] - in[1], b1 = in[2] - in[3], b2 = in[4] - in[5], b3 = in[6] - in[7];
#pragma unroll
    for (int half = 0; half < 2; half++) {
        int e0 = half ? b0 + b3 : a0 + a3, e1 = half ? b1 + b2 : a1 + a2, e2 = half ? b1 - b2 : a1 - a2, e3 = half ? b0 - b3 : a0 - a3;
        if (FAST) {
            int z = fmul8(e2 + e3, 181);
            out[half] = e0 + e1; out[4 + half] = e0 - e1; out[2 + half] = e3 + z; out[6 + half] = e3 - z;
        } else {
            int z = (e2 + e3) * K0541;
            out[half] = rsr(e0 + e1, 4); out[4 + half] = rsr(e0 - e1, 4);
            out[2 + half] = rsr(z + e3 * K0765, 17); out[6 + half] = rsr(z - e2 * K1847, 17);
        }
    }
}
__device__ __forceinline__ void ifast_1d(const int (&in)[8], int (&out)[8])
{
    int s0 = in[0] + in[7], d0 = in[0] - in[7], s1 = in[1] + in[6], d1 = in[1] - in[6];
    int s2 = in[2] + in[5], d2 = in[2] - in[5], s3 = in[3] + in[4], d3 = in[3] - in[4];
    int e0 = s0 + s3, e3 = s0 - s3, e1 = s1 + s2, e2 = s1 - s2;
    out[0] = e0 + e1; out[4] = e0 - e1;
    int z1 = fmul8(e2 + e3, 181);
    out[2] = e3 + z1; out[6] = e3 - z1;
    int p0 = d3 + d2, p1 = d2 + d1, p2 = d1 + d0;
    int z5 = fmul8(p0 - p2, 98), z2 = fmul8(p0, 139) + z5, z4 = fmul8(p2, 334) + z5, z3 = fmul8(p1, 181);
    int z11 = d0 + z3, z13 = d0 - z3;
    out[5] = z13 + z2; out[3] = z13 - z2; out[1] = z11 + z4; out[7] = z11 - z4;
}

// The two passes of the 2-D forward DCT as FDCTDSPContext.fdct runs them on an int16 block (FDCT as in ff_fdct_batch_cuda 0..3, 6, 7):
// fdct_row = the row pass of one row with the int16 write-back the C code does between the passes, fdct_cols = the column pass over a
// block held in registers (not yet truncated: the caller's int16 store does that).  The FAAN transforms (6 ff_faandct, 7 ff_faandct248)
// keep float between the passes (faandct.c's temp[]): their row pass leaves the float's bits in m, and their column pass reads them back.
template <int FDCT>
__device__ __forceinline__ void fdct_row(const int (&in)[8], int (&out)[8])
{
    if constexpr (FDCT >= 6) {
        float t[8];
        faan::fdct_row(in, t);
#pragma unroll
        for (int k = 0; k < 8; k++) out[k] = __float_as_int(t[k]);
        return;
    }
    int o[8];
    if (FDCT < 2) islow_1d<4, 9>(in, o); else ifast_1d(in, o);
#pragma unroll
    for (int k = 0; k < 8; k++) out[k] = (int)(int16_t)o[k];
}
template <int FDCT>
__device__ __forceinline__ void fdct_cols(int (&m)[8][8])
{
#pragma unroll
    for (int c = 0; c < 8; c++) {
        int in[8], o[8];
#pragma unroll
        for (int k = 0; k < 8; k++) in[k] = m[k][c];
        if constexpr (FDCT >= 6) {
            float t[8];
#pragma unroll
            for (int k = 0; k < 8; k++) t[k] = __int_as_float(in[k]);
            if (FDCT == 6) faan::fdct_col(t, c, o); else faan::fdct248_col(t, c, o);
        }
        else if (FDCT == 0) islow_1d<-4, 17>(in, o);
        else if (FDCT == 1) col_248<false>(in, o);
        else if (FDCT == 2) ifast_1d(in, o);
        else col_248<true>(in, o);
#pragma unroll
        for (int k = 0; k < 8; k++) m[k][c] = o[k];
    }
}

// PixblockDSPContext.get_pixels / diff_pixels (pixblockdsp_template.c:24-66) of the 8x8 block at a (minus the one at b, b != NULL),
// optionally followed by the forward DCT in the same thread (FDCT as in ff_fdct_batch_cuda 0..3, 6, 7; < 0: the samples / differences): the
// spatial block never exists as int16 in memory.  m holds what the C code leaves in its int16 block (the column pass is not yet truncated).
// Shared by pixblock_kernel (me_cmp.cu) and the quantiser's front end (mpv_quant.cu).
template <int FDCT>
__device__ __forceinline__ void pixblock_fetch(const uint8_t *a, const uint8_t *b, ptrdiff_t stride, int (&m)[8][8])
{
    const bool vec = !(((uintptr_t)a | (uintptr_t)b | (uintptr_t)stride) & 7);
#pragma unroll
    for (int r = 0; r < 8; r++) {
        int in[8];
        if (vec) {
            const uint2 pa = *reinterpret_cast<const uint2 *>(a + r * stride);
#pragma unroll
            for (int k = 0; k < 4; k++) { in[k] = byte_of(pa.x, k); in[4 + k] = byte_of(pa.y, k); }
            if (b) {
                const uint2 pb = *reinterpret_cast<const uint2 *>(b + r * stride);
#pragma unroll
                for (int k = 0; k < 4; k++) { in[k] -= byte_of(pb.x, k); in[4 + k] -= byte_of(pb.y, k); }
            }
        } else {
#pragma unroll
            for (int k = 0; k < 8; k++) in[k] = a[r * stride + k] - (b ? b[r * stride + k] : 0);
        }
        if (FDCT < 0) {
#pragma unroll
            for (int k = 0; k < 8; k++) m[r][k] = in[k];
        } else fdct_row<FDCT>(in, m[r]);
    }
    if (FDCT >= 0) fdct_cols<FDCT>(m);
}

// the forward DCT of an int16 block in memory (16-byte aligned), into registers as pixblock_fetch leaves them
template <int FDCT>
__device__ __forceinline__ void fdct_load(const int16_t *b, int (&m)[8][8])
{
#pragma unroll
    for (int r = 0; r < 8; r++) {
        const uint4 v = reinterpret_cast<const uint4 *>(b)[r];
        const int in[8] = { lo16s(v.x), hi16s(v.x), lo16s(v.y), hi16s(v.y), lo16s(v.z), hi16s(v.z), lo16s(v.w), hi16s(v.w) };
        fdct_row<FDCT>(in, m[r]);
    }
    fdct_cols<FDCT>(m);
}

}  // namespace avb
