// libav_b200/csrc/fdct10.cu -- the 10-bit instances of the accurate integer forward DCT: ff_jpeg_fdct_islow_10 / ff_fdct248_islow_10
// (libavcodec/jfdctint_template.c with BIT_DEPTH 10: CONST_BITS 13, PASS1_BITS 1, OUT_SHIFT 2, :126-130), what ff_fdctdsp_init() installs
// for bits_per_raw_sample == 10 (fdctdsp.c:31-33).  One thread transforms one block in place (rows with int16 write-back, then columns);
// the passes are in fdct10.cuh, which the ProRes encoder shares.  Reached through ff_fdct_batch_cuda(which = 4 | 5, ...) and the
// FDCTDSPContext slots.  Two kernels with the same arithmetic: the batched one stages a warp's 32 blocks through shared memory (block_stage.cuh: coalesced 512-byte requests in and out, 256 B of traffic per block);
// the thread-per-block one serves unaligned block arrays and tests/hostsim/ (its threads never communicate).
#include "common.cuh"
#include "fdct10.cuh"
#ifndef AVB_HOSTSIM
#include "block_stage.cuh"
#endif

namespace avb {

__global__ void __launch_bounds__(128) fdct10_kernel(int is248, int16_t *__restrict__ blocks, size_t n)
{
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    int16_t *g = blocks + 64 * i;
    int16_t b[64];
    for (int k = 0; k < 64; k++) b[k] = g[k];
    int in[8], out[8];
    for (int r = 0; r < 8; r++) {                          // PASS1_BITS 1: rows scaled up by 2, descaled by CONST_BITS - PASS1_BITS = 12
        for (int k = 0; k < 8; k++) in[k] = b[8 * r + k];
        f10_islow_1d(in, out, 1, 12);
        for (int k = 0; k < 8; k++) b[8 * r + k] = (int16_t)out[k];
    }
    for (int c = 0; c < 8; c++) {                          // OUT_SHIFT 2
        for (int k = 0; k < 8; k++) in[k] = b[8 * k + c];
        if (is248) f10_248_col(in, out, 2, 15); else f10_islow_1d(in, out, -2, 15);
        for (int k = 0; k < 8; k++) g[8 * k + c] = (int16_t)out[k];
    }
}

#ifndef AVB_HOSTSIM
constexpr int F10_WARPS = 4;
__global__ void __launch_bounds__(F10_WARPS * 32) fdct10_staged_kernel(int is248, int16_t *__restrict__ blocks, size_t n)
{
    __shared__ __align__(128) uint4 tile[F10_WARPS][2][256];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const WarpBlockStage S(&tile[warp][0][0], lane);
    const size_t groups = (n + 31) / 32, gstride = (size_t)gridDim.x * F10_WARPS;
    size_t g = (size_t)blockIdx.x * F10_WARPS + warp;
    unsigned buf = 0;
    if (g < groups) S.issue(blocks, g, n, S.buffer(0));
    for (; g < groups; g += gstride, buf ^= 4096u) {
        const size_t gn = g + gstride;
        const unsigned tb = S.buffer(buf);
        if (gn < groups) { S.issue(blocks, gn, n, S.buffer(buf ^ 4096u)); cp_async_wait<1>(); } else cp_async_wait<0>();
        __syncwarp();
        uint32_t m[8][4];                                  // the block after the row pass, int16 pairs
#pragma unroll
        for (int r = 0; r < 8; r++) {
            const uint4 v = S.row(tb, r);
            const int in[8] = { lo16s(v.x), hi16s(v.x), lo16s(v.y), hi16s(v.y), lo16s(v.z), hi16s(v.z), lo16s(v.w), hi16s(v.w) };
            int o[8];
            f10_islow_1d(in, o, 1, 12);
            m[r][0] = pack16(o[0], o[1]); m[r][1] = pack16(o[2], o[3]); m[r][2] = pack16(o[4], o[5]); m[r][3] = pack16(o[6], o[7]);
        }
        uint32_t res[8][4];
#pragma unroll
        for (int c = 0; c < 4; c++) {
            int lo[8], hi[8], olo[8], ohi[8];
#pragma unroll
            for (int k = 0; k < 8; k++) { lo[k] = lo16s(m[k][c]); hi[k] = hi16s(m[k][c]); }
            if (is248) { f10_248_col(lo, olo, 2, 15); f10_248_col(hi, ohi, 2, 15); }
            else       { f10_islow_1d(lo, olo, -2, 15); f10_islow_1d(hi, ohi, -2, 15); }
#pragma unroll
            for (int k = 0; k < 8; k++) res[k][c] = pack16(olo[k], ohi[k]);
        }
#pragma unroll
        for (int r = 0; r < 8; r++) S.put_row(tb, r, make_uint4(res[r][0], res[r][1], res[r][2], res[r][3]));
        S.flush(blocks, g, n, tb);
        __syncwarp();
    }
}
#endif

// which 4 = jpeg_fdct_islow_10, 5 = fdct248_islow_10 (the numbering of ff_fdct_batch_cuda)
int fdct10_launch(int which, int16_t *blocks, size_t n, cudaStream_t st)
{
    if (!n) return 0;
#ifndef AVB_HOSTSIM
    if (!((uintptr_t)blocks & 15)) {
        const size_t groups = (n + 31) / 32;
        const unsigned grid = (unsigned)min((size_t)sm_count() * 8, (groups + F10_WARPS - 1) / F10_WARPS);
        fdct10_staged_kernel<<<grid, F10_WARPS * 32, 0, st>>>(which == 5, blocks, n);
        return check_launch("fdct_batch (10 bit)");
    }
#endif
    AVB_LAUNCH(fdct10_kernel, dim3((unsigned)((n + 127) / 128)), dim3(128), 0, st)(which == 5, blocks, n);
    return check_launch("fdct_batch (10 bit)");
}

}  // namespace avb
