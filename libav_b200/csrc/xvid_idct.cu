// libav_b200/csrc/xvid_idct.cu -- the Xvid IDCT: ff_xvid_idct / xvid_idct_put / xvid_idct_add (libavcodec/xvididct.c:272-331), what
// ff_xvid_idct_init() installs for MPEG-4 streams written by Xvid (and for idct_algo FF_IDCT_XVID), as a batched entry point, fused behind
// the inverse quantisers, and as the three table slots (a batch of one).
//
// The batched path is the 8-bit IDCT kernel of idctdsp.cu with the Xvid transform policy (xvid_idct.cuh): same staging, TMA / cp.async
// fetch, addressing, fused clear and dequantisation.  That kernel needs 16-byte aligned blocks and 8-byte aligned destination rows; any
// other batch runs the thread-per-block kernel below, whose threads never communicate, so the file also compiles for tests/hostsim/.
#include "common.cuh"
#include "scratch.h"
#include "idct_dq.h"
#include "xvid_idct.cuh"
#include "../../include/avdsp_b200.h"
#include <string.h>

namespace avb {

#ifndef AVB_HOSTSIM
int launch_xvid_idct_staged(int mode, int16_t *blocks, uint8_t *frame, const uint32_t *dst_off, ptrdiff_t stride,
                            size_t n, int tiles_per_row, int clear, cudaStream_t st);
int launch_mpeg_dequant_xvid_idct(int kind, const DqTables &t, const uint32_t *recs, int16_t *blocks, uint8_t *frame,
                                  const uint32_t *dst_off, ptrdiff_t stride, size_t n, int tiles_per_row, int clear, cudaStream_t st);
#endif

// one thread per block, 2-byte accesses throughout: mode 0 put, 1 add, 2 in place; `clear` zeroes a put / add block afterwards
__global__ void __launch_bounds__(128) xvid_idct_block_kernel(int mode, int clear, int16_t *blocks, uint8_t *frame, const uint32_t *dst_off,
                                                              ptrdiff_t stride, size_t n, int tiles_per_row)
{
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    int16_t *g = blocks + 64 * i;
    uint4 row[8];
    for (int r = 0; r < 8; r++) {
        const int16_t *s = g + 8 * r;
        row[r] = xvid_row(make_uint4(pack16(s[0], s[1]), pack16(s[2], s[3]), pack16(s[4], s[5]), pack16(s[6], s[7])), r);
    }
    uint8_t *dst = nullptr;
    if (mode != 2) {
        const size_t ty = dst_off ? 0 : i / (unsigned)tiles_per_row;
        dst = frame + (dst_off ? (size_t)dst_off[i] : ty * 8 * (size_t)stride + (i - ty * (unsigned)tiles_per_row) * 8);
    }
    for (int c = 0; c < 4; c++) {
        uint32_t w[8];
        for (int r = 0; r < 8; r++) w[r] = c == 0 ? row[r].x : c == 1 ? row[r].y : c == 2 ? row[r].z : row[r].w;
        int v[2][8];
        XvidIdct::col<0, false>(w, v[0]);
        XvidIdct::col<1, false>(w, v[1]);
        for (int y = 0; y < 8; y++)
            for (int h = 0; h < 2; h++) {
                if (mode == 2) { g[8 * y + 2 * c + h] = (int16_t)v[h][y]; continue; }
                uint8_t *p = dst + y * stride + 2 * c + h;
                *p = (uint8_t)clip_u8(v[h][y] + (mode == 1 ? *p : 0));
            }
    }
    if (mode != 2 && clear)
        for (int k = 0; k < 64; k++) g[k] = 0;
}

static int launch_xvid_idct(int mode, int16_t *blocks, uint8_t *frame, const uint32_t *dst_off, ptrdiff_t stride, size_t n,
                            int tiles_per_row, int clear, cudaStream_t st)
{
    if (n == 0) return 0;
    if (mode < 0 || mode > 2 || !blocks || (mode != 2 && !frame)) { set_error_msg("xvid_idct_batch", "bad mode / pointer"); return -1; }
    if (mode != 2 && !dst_off && tiles_per_row <= 0) { set_error_msg("xvid_idct_batch", "need dst_off or tiles_per_row"); return -1; }
#ifndef AVB_HOSTSIM
    if (!((uintptr_t)blocks & 15) && (mode == 2 || !(((uintptr_t)frame | (uintptr_t)stride) & 7)))
        return launch_xvid_idct_staged(mode, blocks, frame, dst_off, stride, n, tiles_per_row, clear, st);
#endif
    AVB_LAUNCH(xvid_idct_block_kernel, dim3((unsigned)((n + 127) / 128)), dim3(128), 0, st)(mode, clear, blocks, frame, dst_off, stride, n, tiles_per_row);
    return check_launch("xvid_idct_batch");
}

namespace {

// table slots: a batch of one with host pointers.  Device layout: [0,128) the block, [128,192) the 8 x 8 pixels at pitch 8.
template <int MODE> void slot_xvid(uint8_t *dest, ptrdiff_t line_size, int16_t *block)
{
    ScratchLock lk;
    Scratch &S = scratch();
    uint8_t *h = (uint8_t *)S.pinned(256), *d = (uint8_t *)S.dev(3, 256);
    cudaStream_t *st = S.streams();
    if (!h || !d || !st) return;
    memcpy(h, block, 128);
    if (MODE == 1) for (int y = 0; y < 8; y++) memcpy(h + 128 + 8 * y, dest + y * line_size, 8);
    if (cudaMemcpyAsync(d, h, MODE == 1 ? 192 : 128, cudaMemcpyHostToDevice, st[0]) != cudaSuccess) { set_error("xvid slot:h2d", cudaGetLastError()); return; }
    if (launch_xvid_idct(MODE, (int16_t *)d, d + 128, nullptr, 8, 1, 1, 0, st[0])) return;
    if (cudaMemcpyAsync(h, d, 192, cudaMemcpyDeviceToHost, st[0]) != cudaSuccess || cudaStreamSynchronize(st[0]) != cudaSuccess) {
        set_error("xvid slot:d2h", cudaGetLastError()); return;
    }
    if (MODE == 2) memcpy(block, h, 128);
    else for (int y = 0; y < 8; y++) memcpy(dest + y * line_size, h + 128 + 8 * y, 8);
}
void slot_xvid_inplace(int16_t *block) { slot_xvid<2>(nullptr, 0, block); }

}  // namespace

// the three transform entries of ff_xvid_idct_init (xvididct.c:333-350) with FF_IDCT_PERM_NONE
void xvid_idct_install(IDCTDSPContext *c)
{
    c->idct_put = slot_xvid<0>; c->idct_add = slot_xvid<1>; c->idct = slot_xvid_inplace;
    c->perm_type = FF_IDCT_PERM_NONE;
    for (int i = 0; i < 64; i++) c->idct_permutation[i] = (uint8_t)i;     // what ff_init_scantable_permutation() makes of PERM_NONE
}

}  // namespace avb

using namespace avb;

extern "C" {

int ff_xvid_idct_batch_cuda(int mode, int16_t *blocks, uint8_t *frame, const uint32_t *dst_off, ptrdiff_t stride, size_t n,
                            int tiles_per_row, int clear, void *stream)
{
    avb::enter();
    return launch_xvid_idct(mode, blocks, frame, dst_off, stride, n, tiles_per_row, clear, (cudaStream_t)stream);
}

void ff_xvid_idct_init_cuda(IDCTDSPContext *c, int idct_algo, int bits_per_raw_sample)
{
    avb::enter();
    if (!c || bits_per_raw_sample > 8) return;                           // ff_xvid_idct_init declines high bit depth
    if (idct_algo == AVB_FF_IDCT_AUTO || idct_algo == AVB_FF_IDCT_XVID) xvid_idct_install(c);
}

}  // extern "C"
