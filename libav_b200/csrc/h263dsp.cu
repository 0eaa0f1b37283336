// libav_b200/csrc/h263dsp.cu -- the H263DSPContext slots (libavcodec/h263dsp.c:31-124) and their ff_h263dsp_init_cuda hook.
//
// A slot has the C slot's signature and HOST pointers.  It stages the 4 x 8 samples the C function reads and writes around src (two
// before it), runs the slot kernel of h263_lf.cuh -- the picture filter's line arithmetic, one thread per line -- on them, writes them
// back and synchronises.  The drop-in path; decoders that flush whole pictures use ff_h263_loop_filter_batch_cuda.
#include "h263_lf.cuh"
#include "scratch.h"
#include "../../include/avdsp_b200.h"

namespace avb {

namespace {

constexpr int SP = 8;      // pitch of the staged rectangle

// vert 1: h263_h_loop_filter (columns -2 .. 1 of 8 rows); vert 0: h263_v_loop_filter (rows -2 .. 1 of 8 columns)
template <int VERT> void slot_h263_loop_filter(uint8_t *src, int stride, int qscale)
{
    if (qscale < 0 || qscale > 31) return;
    ScratchLock lk;
    Scratch &S = scratch();
    uint8_t *h = (uint8_t *)S.pinned2(64), *d = (uint8_t *)S.dev(4, 64);
    cudaStream_t *st = S.streams();
    if (!h || !d || !st) return;
    const int w = VERT ? 4 : 8, rows = VERT ? 8 : 4;
    uint8_t *org = VERT ? src - 2 : src - 2 * (ptrdiff_t)stride;
    for (int y = 0; y < rows; y++) memcpy(h + y * SP, org + (ptrdiff_t)y * stride, w);
    if (cudaMemcpyAsync(d, h, rows * SP, cudaMemcpyHostToDevice, st[0]) != cudaSuccess) { set_error("h263 loop filter slot:h2d", cudaGetLastError()); return; }
    AVB_LAUNCH(h263_lf_slot_kernel, 1, 32, 0, st[0])(VERT ? d + 2 : d + 2 * SP, SP, (int)h263_lf_strength_tab[qscale], VERT);
    if (check_launch("h263 loop filter slot")) return;
    if (cudaMemcpyAsync(h, d, rows * SP, cudaMemcpyDeviceToHost, st[0]) != cudaSuccess || cudaStreamSynchronize(st[0]) != cudaSuccess) {
        set_error("h263 loop filter slot:d2h", cudaGetLastError());
        return;
    }
    for (int y = 0; y < rows; y++) memcpy(org + (ptrdiff_t)y * stride, h + y * SP, w);
}

}  // namespace

}  // namespace avb

extern "C" void ff_h263dsp_init_cuda(H263DSPContext *c)
{
    if (!c) return;
    c->h263_h_loop_filter = avb::slot_h263_loop_filter<1>;
    c->h263_v_loop_filter = avb::slot_h263_loop_filter<0>;
}
