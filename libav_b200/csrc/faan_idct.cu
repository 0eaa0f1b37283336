// libav_b200/csrc/faan_idct.cu -- the floating-point AAN transforms (faan_dct.cuh): ff_faanidct / _put / _add (libavcodec/faanidct.c:113-159),
// what ff_idctdsp_init() installs for idct_algo FF_IDCT_FAAN, as a batched entry point and as the three table slots (a batch of one); and the
// forward pair ff_faandct / ff_faandct248 (libavcodec/faandct.c:121-215) behind ff_fdct_batch_cuda 6 / 7.
//
// The batched IDCT runs faan_idct_kernel (idctdsp.cu) over the 8-bit IDCT's staging.  That kernel needs 16-byte aligned blocks and 8-byte
// aligned destination rows; any other batch runs the thread-per-block kernel below.  Threads never communicate in this file, so it also
// compiles for tests/hostsim/.
#include "common.cuh"
#include "scratch.h"
#include "fdct_dev.cuh"
#include "faan_dct.cuh"
#include "../../include/avdsp_b200.h"
#include <string.h>

namespace avb {

#ifndef AVB_HOSTSIM
int launch_faan_idct_staged(int mode, int16_t *blocks, uint8_t *frame, const uint32_t *dst_off, ptrdiff_t stride,
                            size_t n, int tiles_per_row, int clear, cudaStream_t st);
#endif

// one thread per block, 2-byte accesses throughout: mode 0 put, 1 add, 2 in place; `clear` zeroes a put / add block afterwards
__global__ void __launch_bounds__(128) faan_idct_block_kernel(int mode, int clear, int16_t *blocks, uint8_t *frame, const uint32_t *dst_off,
                                                              ptrdiff_t stride, size_t n, int tiles_per_row)
{
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    int16_t *g = blocks + 64 * i;
    float t[8][8];
    for (int r = 0; r < 8; r++) {
        int x[8];
        for (int c = 0; c < 8; c++) x[c] = g[8 * r + c];
        faan::idct_row(x, r, t[r]);
    }
    uint8_t *dst = nullptr;
    if (mode != 2) {
        const size_t ty = dst_off ? 0 : i / (unsigned)tiles_per_row;
        dst = frame + (dst_off ? (size_t)dst_off[i] : ty * 8 * (size_t)stride + (i - ty * (unsigned)tiles_per_row) * 8);
    }
    for (int c = 0; c < 8; c++) {
        float col[8];
        for (int k = 0; k < 8; k++) col[k] = t[k][c];
        faan::idct_1d(col);
        for (int y = 0; y < 8; y++) {
            const int v = __float2int_rn(col[y]);
            if (mode == 2) { g[8 * y + c] = (int16_t)v; continue; }
            uint8_t *p = dst + y * stride + c;
            *p = (uint8_t)clip_u8(v + (mode == 1 ? *p : 0));
        }
    }
    if (mode != 2 && clear)
        for (int k = 0; k < 64; k++) g[k] = 0;
}

static int launch_faan_idct(int mode, int16_t *blocks, uint8_t *frame, const uint32_t *dst_off, ptrdiff_t stride, size_t n,
                            int tiles_per_row, int clear, cudaStream_t st)
{
    if (n == 0) return 0;
    if (mode < 0 || mode > 2 || !blocks || (mode != 2 && !frame)) { set_error_msg("faanidct_batch", "bad mode / pointer"); return -1; }
    if (mode != 2 && !dst_off && tiles_per_row <= 0) { set_error_msg("faanidct_batch", "need dst_off or tiles_per_row"); return -1; }
#ifndef AVB_HOSTSIM
    if (!((uintptr_t)blocks & 15) && (mode == 2 || !(((uintptr_t)frame | (uintptr_t)stride) & 7)))
        return launch_faan_idct_staged(mode, blocks, frame, dst_off, stride, n, tiles_per_row, clear, st);
#endif
    AVB_LAUNCH(faan_idct_block_kernel, dim3((unsigned)((n + 127) / 128)), dim3(128), 0, st)(mode, clear, blocks, frame, dst_off, stride, n, tiles_per_row);
    return check_launch("faanidct_batch");
}

// ff_faandct (WHICH 6) / ff_faandct248 (7) in place, one thread per block
template <int WHICH>
__global__ void __launch_bounds__(128) faan_fdct_kernel(int16_t *blocks, size_t n)
{
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    int16_t *b = blocks + 64 * i;
    int m[8][8];
    for (int r = 0; r < 8; r++) {
        int in[8];
        for (int c = 0; c < 8; c++) in[c] = b[8 * r + c];
        fdct_row<WHICH>(in, m[r]);
    }
    fdct_cols<WHICH>(m);
    for (int k = 0; k < 64; k++) b[k] = (int16_t)m[k >> 3][k & 7];
}

// ff_fdct_batch_cuda 6 / 7 (me_cmp.cu); blocks at any 2-byte alignment
int faan_fdct_launch(int which, int16_t *blocks, size_t n, cudaStream_t st)
{
    if (n == 0) return 0;
    const dim3 grid((unsigned)((n + 127) / 128)), block(128);
    if (which == 6) AVB_LAUNCH(faan_fdct_kernel<6>, grid, block, 0, st)(blocks, n);
    else if (which == 7) AVB_LAUNCH(faan_fdct_kernel<7>, grid, block, 0, st)(blocks, n);
    else { set_error_msg("fdct_batch", "bad transform selector"); return -1; }
    return check_launch("fdct_batch");
}

namespace {

// table slots: a batch of one with host pointers.  Device layout: [0,128) the block, [128,192) the 8 x 8 pixels at pitch 8.
template <int MODE> void slot_faan(uint8_t *dest, ptrdiff_t line_size, int16_t *block)
{
    ScratchLock lk;
    Scratch &S = scratch();
    uint8_t *h = (uint8_t *)S.pinned(256), *d = (uint8_t *)S.dev(3, 256);
    cudaStream_t *st = S.streams();
    if (!h || !d || !st) return;
    memcpy(h, block, 128);
    if (MODE == 1) for (int y = 0; y < 8; y++) memcpy(h + 128 + 8 * y, dest + y * line_size, 8);
    if (cudaMemcpyAsync(d, h, MODE == 1 ? 192 : 128, cudaMemcpyHostToDevice, st[0]) != cudaSuccess) { set_error("faan slot:h2d", cudaGetLastError()); return; }
    if (launch_faan_idct(MODE, (int16_t *)d, d + 128, nullptr, 8, 1, 1, 0, st[0])) return;
    if (cudaMemcpyAsync(h, d, 192, cudaMemcpyDeviceToHost, st[0]) != cudaSuccess || cudaStreamSynchronize(st[0]) != cudaSuccess) {
        set_error("faan slot:d2h", cudaGetLastError()); return;
    }
    if (MODE == 2) memcpy(block, h, 128);
    else for (int y = 0; y < 8; y++) memcpy(dest + y * line_size, h + 128 + 8 * y, 8);
}
void slot_faan_inplace(int16_t *block) { slot_faan<2>(nullptr, 0, block); }

}  // namespace

// the three transform entries ff_idctdsp_init gives FF_IDCT_FAAN (idctdsp.c:162-166), with FF_IDCT_PERM_NONE
void faan_idct_install(IDCTDSPContext *c)
{
    c->idct_put = slot_faan<0>; c->idct_add = slot_faan<1>; c->idct = slot_faan_inplace;
    c->perm_type = FF_IDCT_PERM_NONE;
    for (int i = 0; i < 64; i++) c->idct_permutation[i] = (uint8_t)i;     // what ff_init_scantable_permutation() makes of PERM_NONE
}

}  // namespace avb

using namespace avb;

extern "C" int ff_faanidct_batch_cuda(int mode, int16_t *blocks, uint8_t *frame, const uint32_t *dst_off, ptrdiff_t stride, size_t n,
                                      int tiles_per_row, int clear, void *stream)
{
    avb::enter();
    return launch_faan_idct(mode, blocks, frame, dst_off, stride, n, tiles_per_row, clear, (cudaStream_t)stream);
}
