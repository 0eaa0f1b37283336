// libav_b200/csrc/mpegvideodsp.cu -- the MpegVideoDSPContext slots (libavcodec/mpegvideodsp.c:24-119) and their ff_mpegvideodsp_init_cuda
// hook.
//
// A slot has the C slot's signature and HOST pointers.  It stages the samples the C function can read, runs the slot kernel -- the GMC
// arithmetic of mpv_gmc.cuh, one thread per destination sample -- on them, writes the 8 x h block back and synchronises.  The drop-in
// path; decoders that flush whole pictures send S-VOPs through ff_mpv_motion_batch_cuda.
#include "mpv_gmc.cuh"
#include "scratch.h"
#include "../../include/avdsp_b200.h"
#include <climits>

namespace avb {

// what one slot call computes: gmc1_c (kind 0) or ff_gmc_c (kind 1) on a staged rectangle whose sample (0, 0) is source sample (x0, y0)
struct MpvGmcSlot {
    int kind, h, pitch, x0, y0;
    int x16, y16, rounder;                                                  // gmc1_c
    int ox, oy, dxx, dxy, dyx, dyy, shift, r, width, height;               // ff_gmc_c
};

__global__ void __launch_bounds__(128) mpv_gmc_slot_kernel(uint8_t *dst, const uint8_t *src, const MpvGmcSlot a)
{
    const int t = blockIdx.x * blockDim.x + threadIdx.x, x = t & 7, y = t >> 3;
    if (y >= a.h) return;
    const auto f = [&](int xx, int yy) { return (int)src[(ptrdiff_t)(yy - a.y0) * a.pitch + (xx - a.x0)]; };
    int v;
    if (a.kind == 0) {
        v = mpv_gmc1_sample(f, x, y, a.x16, a.y16, a.rounder);
    } else {
        const uint32_t vx = (uint32_t)a.ox + (uint32_t)a.dxx * (uint32_t)x + (uint32_t)a.dxy * (uint32_t)y;
        const uint32_t vy = (uint32_t)a.oy + (uint32_t)a.dyx * (uint32_t)x + (uint32_t)a.dyy * (uint32_t)y;
        v = mpv_gmc_sample(f, vx, vy, a.shift, a.r, a.width, a.height);
    }
    dst[8 * y + x] = (uint8_t)v;
}

namespace {

// stage rows [y0, y0 + rows) x columns [x0, x0 + a.pitch) of the plane at src, run the slot kernel, write the 8 x h block back
void gmc_slot_run(uint8_t *dst, const uint8_t *src, int stride, int rows, MpvGmcSlot a)
{
    if (a.h <= 0) return;
    ScratchLock lk;
    Scratch &S = scratch();
    const size_t in = (size_t)a.pitch * rows, out = (size_t)8 * a.h;
    uint8_t *h = (uint8_t *)S.pinned(in + out), *d = (uint8_t *)S.dev(4, in + out);
    cudaStream_t *st = S.streams();
    if (!h || !d || !st) return;
    for (int y = 0; y < rows; y++) memcpy(h + (size_t)y * a.pitch, src + (ptrdiff_t)(a.y0 + y) * stride + a.x0, a.pitch);
    if (cudaMemcpyAsync(d, h, in, cudaMemcpyHostToDevice, st[0]) != cudaSuccess) { set_error("mpegvideodsp slot:h2d", cudaGetLastError()); return; }
    AVB_LAUNCH(mpv_gmc_slot_kernel, (unsigned)((out + 127) / 128), 128, 0, st[0])(d + in, d, a);
    if (check_launch("mpegvideodsp slot")) return;
    if (cudaMemcpyAsync(h + in, d + in, out, cudaMemcpyDeviceToHost, st[0]) != cudaSuccess || cudaStreamSynchronize(st[0]) != cudaSuccess) {
        set_error("mpegvideodsp slot:d2h", cudaGetLastError());
        return;
    }
    for (int y = 0; y < a.h; y++) memcpy(dst + (ptrdiff_t)y * stride, h + in + 8 * y, 8);
}

// gmc1_c reads the 9 x (h + 1) samples at src
void slot_gmc1(uint8_t *dst, uint8_t *src, int stride, int h, int x16, int y16, int rounder)
{
    MpvGmcSlot a = {};
    a.kind = 0; a.h = h; a.pitch = 9; a.x16 = x16; a.y16 = y16; a.rounder = rounder;
    gmc_slot_run(dst, src, stride, h + 1, a);
}

// ff_gmc_c reads inside [0, width) x [0, height): the positions of the block's four corners bound what it reads (the map is affine and the
// shifts and clips are monotone), one more column / row for the bilinear neighbour; a corner outside int32 stages the whole plane
void slot_gmc(uint8_t *dst, uint8_t *src, int stride, int h, int ox, int oy, int dxx, int dxy, int dyx, int dyy, int shift, int r,
              int width, int height)
{
    if (h <= 0 || width <= 0 || height <= 0 || shift < 0 || shift > 15) return;
    long long lo[2] = { LLONG_MAX, LLONG_MAX }, hi[2] = { LLONG_MIN, LLONG_MIN };
    bool whole = false;
    for (int cy = 0; cy < 2; cy++)
        for (int cx = 0; cx < 2; cx++) {
            const long long x = 7 * cx, y = (long long)(h - 1) * cy;
            const long long v[2] = { (long long)ox + dxx * x + dxy * y, (long long)oy + dyx * x + dyy * y };
            for (int k = 0; k < 2; k++) {
                if (v[k] < INT_MIN || v[k] > INT_MAX) whole = true;
                const long long p = v[k] >> (16 + shift);
                lo[k] = p < lo[k] ? p : lo[k];
                hi[k] = p > hi[k] ? p : hi[k];
            }
        }
    const long long ext[2] = { width, height };
    long long a0[2], a1[2];
    for (int k = 0; k < 2; k++) {
        a0[k] = whole ? 0 : lo[k] < 0 ? 0 : lo[k] > ext[k] - 1 ? ext[k] - 1 : lo[k];
        a1[k] = whole ? ext[k] - 1 : hi[k] + 1 < 0 ? 0 : hi[k] + 1 > ext[k] - 1 ? ext[k] - 1 : hi[k] + 1;
    }
    MpvGmcSlot a = {};
    a.kind = 1; a.h = h; a.x0 = (int)a0[0]; a.y0 = (int)a0[1]; a.pitch = (int)(a1[0] - a0[0] + 1);
    a.ox = ox; a.oy = oy; a.dxx = dxx; a.dxy = dxy; a.dyx = dyx; a.dyy = dyy; a.shift = shift; a.r = r; a.width = width; a.height = height;
    gmc_slot_run(dst, src, stride, (int)(a1[1] - a0[1] + 1), a);
}

}  // namespace

}  // namespace avb

extern "C" void ff_mpegvideodsp_init_cuda(MpegVideoDSPContext *c)
{
    if (!c) return;
    c->gmc1 = avb::slot_gmc1;
    c->gmc = avb::slot_gmc;
}
