// libav_b200/csrc/idct10.cu -- the 10-bit instance of the simple IDCT: ff_simple_idct_put_10 / _add_10 / _10
// (libavcodec/simple_idct_template.c with BIT_DEPTH 10, :63-78: 17-bit constants, ROW_SHIFT 15, COL_SHIFT 20, DC_SHIFT 1; 16-bit
// samples clipped to 10 bits), what ff_idctdsp_init() installs for bits_per_raw_sample == 10 (idctdsp.c:151-155).
// One thread transforms one block (both passes in registers / local memory, the block array is left exactly as the C functions
// leave it: row-pass intermediates for put / add, the result for the in-place call).  This is the functional path for 10-bit
// content -- a batched entry point plus the three table slots as a batch of one; it has not been tuned like the 8-bit kernel
// (idctdsp.cu).  Threads never communicate: the file also compiles for tests/hostsim/.
#include "common.cuh"
#include "scratch.h"
#ifndef AVB_HOSTSIM
#include "block_stage.cuh"
#include "idct10.cuh"
#endif
#include "../../include/avdsp_b200.h"
#include <string.h>

namespace avb {

__device__ inline void idct10_rows(int16_t *b)
{
    constexpr int W1 = 90901, W2 = 85627, W3 = 77062, W4 = 65535, W5 = 51491, W6 = 35468, W7 = 18081;
    for (int r = 0; r < 8; r++) {
        int16_t *row = b + 8 * r;
        if (!(row[1] | row[2] | row[3] | row[4] | row[5] | row[6] | row[7])) {          // DC-only row: row[0] << DC_SHIFT, :94-106
            const int16_t v = (int16_t)((row[0] * 2) & 0xffff);
            for (int k = 0; k < 8; k++) row[k] = v;
            continue;
        }
        int a0 = W4 * row[0] + (1 << 14), a1 = a0, a2 = a0, a3 = a0;
        a0 += W2 * row[2]; a1 += W6 * row[2]; a2 -= W6 * row[2]; a3 -= W2 * row[2];
        int b0 = W1 * row[1] + W3 * row[3], b1 = W3 * row[1] - W7 * row[3], b2 = W5 * row[1] - W1 * row[3], b3 = W7 * row[1] - W5 * row[3];
        if (row[4] | row[5] | row[6] | row[7]) {
            a0 += W4 * row[4] + W6 * row[6]; a1 += -W4 * row[4] - W2 * row[6]; a2 += -W4 * row[4] + W2 * row[6]; a3 += W4 * row[4] - W6 * row[6];
            b0 += W5 * row[5] + W7 * row[7]; b1 += -W1 * row[5] - W5 * row[7]; b2 += W7 * row[5] + W3 * row[7]; b3 += W3 * row[5] - W1 * row[7];
        }
        row[0] = (int16_t)((a0 + b0) >> 15); row[7] = (int16_t)((a0 - b0) >> 15); row[1] = (int16_t)((a1 + b1) >> 15); row[6] = (int16_t)((a1 - b1) >> 15);
        row[2] = (int16_t)((a2 + b2) >> 15); row[5] = (int16_t)((a2 - b2) >> 15); row[3] = (int16_t)((a3 + b3) >> 15); row[4] = (int16_t)((a3 - b3) >> 15);
    }
}
__device__ inline void idct10_col(const int16_t *col, int (&out)[8])
{
    constexpr int W1 = 90901, W2 = 85627, W3 = 77062, W4 = 65535, W5 = 51491, W6 = 35468, W7 = 18081;
    int a0 = W4 * (col[0] + ((1 << 19) / W4)), a1 = a0, a2 = a0, a3 = a0;             // rounding folded into the DC term, :176
    a0 += W2 * col[16]; a1 += W6 * col[16]; a2 -= W6 * col[16]; a3 -= W2 * col[16];
    int b0 = W1 * col[8] + W3 * col[24], b1 = W3 * col[8] - W7 * col[24], b2 = W5 * col[8] - W1 * col[24], b3 = W7 * col[8] - W5 * col[24];
    a0 += W4 * col[32]; a1 -= W4 * col[32]; a2 -= W4 * col[32]; a3 += W4 * col[32];
    b0 += W5 * col[40]; b1 -= W1 * col[40]; b2 += W7 * col[40]; b3 += W3 * col[40];
    a0 += W6 * col[48]; a1 -= W2 * col[48]; a2 += W2 * col[48]; a3 -= W6 * col[48];
    b0 += W7 * col[56]; b1 -= W5 * col[56]; b2 += W3 * col[56]; b3 -= W1 * col[56];
    out[0] = (a0 + b0) >> 20; out[1] = (a1 + b1) >> 20; out[2] = (a2 + b2) >> 20; out[3] = (a3 + b3) >> 20;
    out[4] = (a3 - b3) >> 20; out[5] = (a2 - b2) >> 20; out[6] = (a1 - b1) >> 20; out[7] = (a0 - b0) >> 20;
}

// mode 0 put, 1 add, 2 in place; block i -> frame + dst_off[i] (bytes), rows stride_px samples apart
__global__ void __launch_bounds__(128) simple_idct10_kernel(int mode, int16_t *__restrict__ blocks, uint16_t *frame, const uint32_t *__restrict__ dst_off,
                                                            ptrdiff_t stride_px, size_t n)
{
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    int16_t b[64];
    int16_t *g = blocks + 64 * i;
    for (int k = 0; k < 64; k++) b[k] = g[k];
    idct10_rows(b);
    if (mode != 2) for (int k = 0; k < 64; k++) g[k] = b[k];          // the C functions leave the row-pass intermediates in the block
    uint16_t *d = mode == 2 ? nullptr : (uint16_t *)((uint8_t *)frame + dst_off[i]);
    for (int c = 0; c < 8; c++) {
        int o[8];
        idct10_col(b + c, o);
        for (int k = 0; k < 8; k++) {
            if (mode == 2) { g[c + 8 * k] = (int16_t)o[k]; continue; }
            const int v = mode == 1 ? d[c + k * stride_px] + o[k] : o[k];
            d[c + k * stride_px] = (uint16_t)min(max(v, 0), 1023);
        }
    }
}

#ifndef AVB_HOSTSIM
// ---- the batched kernel: the 8-bit kernel's staged layout (idctdsp.cu) ---------------------------------------------------------------
// A warp owns 32 consecutive blocks (4 KB): eight coalesced 512-byte cp.async requests (LDGSTS) bring them into a 128-byte-row XOR-swizzled
// shared-memory tile (double-buffered, the next group in flight), every lane reads ITS block's eight rows as conflict-free LDS.128, both
// passes run in registers.  put / add: the row-pass intermediates go back through the same tile and leave as eight coalesced 512-byte
// stores (the C functions leave them in the block), the 8 x 8 samples leave as eight 16-byte rows per lane (a raster of tiles makes a warp's
// row 512 contiguous bytes).  Algorithmic traffic: 128 B in + 128 B back + 128 B of samples = 384 B per block (in place: 256 B).
namespace {

constexpr int I10_WARPS = 4;

template <int MODE>
__global__ void __launch_bounds__(I10_WARPS * 32)
simple_idct10_staged_kernel(int16_t *__restrict__ blocks, uint8_t *__restrict__ frame, const uint32_t *__restrict__ dst_off, ptrdiff_t stride, size_t n)
{
    __shared__ __align__(128) uint4 tile[I10_WARPS][2][256];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const WarpBlockStage S(&tile[warp][0][0], lane);
    const size_t groups = (n + 31) / 32, gstride = (size_t)gridDim.x * I10_WARPS;
    size_t g = (size_t)blockIdx.x * I10_WARPS + warp;
    unsigned buf = 0;
    if (g < groups) S.issue(blocks, g, n, S.buffer(0));
    for (; g < groups; g += gstride, buf ^= 4096u) {
        const size_t gn = g + gstride;
        const unsigned tb = S.buffer(buf);
        if (gn < groups) { S.issue(blocks, gn, n, S.buffer(buf ^ 4096u)); cp_async_wait<1>(); } else cp_async_wait<0>();
        __syncwarp();
        const size_t i = g * 32 + lane;
        const bool live = i < n;
        uint4 row[8];
#pragma unroll
        for (int r = 0; r < 8; r++) row[r] = i10_row(S.row(tb, r));
        if (MODE != 2) {
            // the row pass goes back over the coefficients (what the C functions leave there)
#pragma unroll
            for (int r = 0; r < 8; r++) S.put_row(tb, r, row[r]);
            S.flush(blocks, g, n, tb);
        }
        uint8_t *dst = MODE == 2 ? nullptr : frame + (live ? dst_off[i] : 0);
        const bool vec = !((uintptr_t)dst & 15);                          // (the pitch is a multiple of 16 here; an odd offset takes sample stores)
        uint4 px[8];
        if (MODE == 1 && live) {
#pragma unroll
            for (int y = 0; y < 8; y++) {
                if (vec) px[y] = *reinterpret_cast<const uint4 *>(dst + y * stride);
                else {
                    const uint16_t *q = reinterpret_cast<const uint16_t *>(dst + y * stride);
                    px[y] = make_uint4(q[0] | (uint32_t)q[1] << 16, q[2] | (uint32_t)q[3] << 16, q[4] | (uint32_t)q[5] << 16, q[6] | (uint32_t)q[7] << 16);
                }
            }
        }
        uint32_t o[8][4];
#pragma unroll
        for (int c = 0; c < 4; c++) {
            uint32_t w[8];
#pragma unroll
            for (int r = 0; r < 8; r++) w[r] = c == 0 ? row[r].x : c == 1 ? row[r].y : c == 2 ? row[r].z : row[r].w;
            int lo[8], hi[8];
            i10_col<0>(w, lo);
            i10_col<1>(w, hi);
#pragma unroll
            for (int y = 0; y < 8; y++) {
                if (MODE == 2) o[y][c] = pack16(lo[y], hi[y]);
                else {
                    const uint32_t p = MODE == 1 ? (c == 0 ? px[y].x : c == 1 ? px[y].y : c == 2 ? px[y].z : px[y].w) : 0u;
                    o[y][c] = (uint32_t)i10_clip(lo[y] + (int)(p & 0xffffu)) | (uint32_t)i10_clip(hi[y] + (int)(p >> 16)) << 16;
                }
            }
        }
        if (MODE == 2) {
            // in place: the result replaces the coefficients
#pragma unroll
            for (int y = 0; y < 8; y++) S.put_row(tb, y, make_uint4(o[y][0], o[y][1], o[y][2], o[y][3]));
            S.flush(blocks, g, n, tb);
        } else if (live) {
#pragma unroll
            for (int y = 0; y < 8; y++) {
                if (vec) *reinterpret_cast<uint4 *>(dst + y * stride) = make_uint4(o[y][0], o[y][1], o[y][2], o[y][3]);
                else {
                    uint16_t *q = reinterpret_cast<uint16_t *>(dst + y * stride);
#pragma unroll
                    for (int c = 0; c < 4; c++) { q[2 * c] = (uint16_t)o[y][c]; q[2 * c + 1] = (uint16_t)(o[y][c] >> 16); }
                }
            }
        }
        __syncwarp();     // every lane is done with this buffer before the next group is requested into it
    }
}

}  // namespace
#endif

// the staged kernel needs 16-byte aligned blocks and, for put / add, a pitch that keeps 16-byte alignment from row to row (a block whose
// offset breaks it stores sample by sample inside the kernel); anything else runs the thread-per-block kernel
static int launch_idct10(int mode, int16_t *blocks, uint8_t *frame, const uint32_t *dst_off, ptrdiff_t stride, size_t n, cudaStream_t st)
{
    if (!n) return 0;
#ifndef AVB_HOSTSIM
    if (!((uintptr_t)blocks & 15) && (mode == 2 || !((uintptr_t)stride & 15))) {
        const size_t groups = (n + 31) / 32;
        const unsigned grid = (unsigned)min((size_t)sm_count() * 8, (groups + I10_WARPS - 1) / I10_WARPS);
        if (mode == 0)      simple_idct10_staged_kernel<0><<<grid, I10_WARPS * 32, 0, st>>>(blocks, frame, dst_off, stride, n);
        else if (mode == 1) simple_idct10_staged_kernel<1><<<grid, I10_WARPS * 32, 0, st>>>(blocks, frame, dst_off, stride, n);
        else                simple_idct10_staged_kernel<2><<<grid, I10_WARPS * 32, 0, st>>>(blocks, frame, dst_off, stride, n);
        return check_launch("ff_simple_idct10_batch_cuda");
    }
#endif
    AVB_LAUNCH(simple_idct10_kernel, dim3((unsigned)((n + 127) / 128)), dim3(128), 0, st)(mode, blocks, (uint16_t *)frame, dst_off, stride / 2, n);
    return check_launch("ff_simple_idct10_batch_cuda");
}

namespace {

// table slots: a batch of one with host pointers
template <int MODE> void slot_idct10(uint8_t *dest, ptrdiff_t line_size, int16_t *block)
{
    ScratchLock lk;
    Scratch &S = scratch();
    uint8_t *h = (uint8_t *)S.pinned2(4096), *d = (uint8_t *)S.dev(8, 4096);
    cudaStream_t *st = S.streams();
    if (!h || !d || !st) return;
    // layout: [0,128) block, [128,132) offset, [256, 256 + 8 * 16) the 8 x 8 samples at pitch 16 bytes
    memcpy(h, block, 128);
    const uint32_t off = 256;
    memcpy(h + 128, &off, 4);
    if (MODE != 2) for (int y = 0; y < 8; y++) memcpy(h + 256 + 16 * y, dest + y * line_size, 16);
    if (cudaMemcpyAsync(d, h, 384, cudaMemcpyHostToDevice, st[0]) != cudaSuccess) { set_error("idct10 slot:h2d", cudaGetLastError()); return; }
    if (launch_idct10(MODE, (int16_t *)d, d, (const uint32_t *)(d + 128), 16, 1, st[0])) return;
    if (cudaMemcpyAsync(h, d, 384, cudaMemcpyDeviceToHost, st[0]) != cudaSuccess || cudaStreamSynchronize(st[0]) != cudaSuccess) { set_error("idct10 slot:d2h", cudaGetLastError()); return; }
    memcpy(block, h, 128);
    if (MODE != 2) for (int y = 0; y < 8; y++) memcpy(dest + y * line_size, h + 256 + 16 * y, 16);
}
void slot_idct10_inplace(int16_t *block) { slot_idct10<2>(nullptr, 0, block); }

}  // namespace

// ff_idctdsp_init_cuda (capi_idct.cu) for bits_per_raw_sample == 10: the three transform entries, FF_IDCT_PERM_NONE (idctdsp.c:151-155)
void idct10_install(IDCTDSPContext *c)
{
    c->idct_put = slot_idct10<0>; c->idct_add = slot_idct10<1>; c->idct = slot_idct10_inplace;
    c->perm_type = FF_IDCT_PERM_NONE;
    for (int i = 0; i < 64; i++) c->idct_permutation[i] = (uint8_t)i;
}

}  // namespace avb

using namespace avb;

extern "C" int ff_simple_idct10_batch_cuda(int mode, int16_t *blocks, uint8_t *frame, const uint32_t *dst_off, ptrdiff_t stride, size_t n, void *stream)
{
    avb::enter();
    if (mode < 0 || mode > 2 || (n && !blocks) || (mode != 2 && n && (!frame || !dst_off)) || (stride & 1)) {
        set_error_msg("ff_simple_idct10_batch_cuda", "bad argument"); return -1;
    }
    return launch_idct10(mode, blocks, frame, dst_off, stride, n, (cudaStream_t)stream);
}
