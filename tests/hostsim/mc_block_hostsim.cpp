// tests/hostsim/mc_block_hostsim.cpp -- TEST INFRASTRUCTURE, NOT PRODUCT.
//
// libav_b200/csrc/h264_mc_block.cuh compiled for the host: mc_block() is the whole arithmetic of the batched H.264 inter prediction (one
// thread = one 4x4 luma block + its 2x2 chroma blocks, no shared memory, no warp collectives), so the CPU suite can run it block after
// block over the same record lists the GPU tests use and compare with the compiled reference.  The work distribution of h264_mc.cu
// (shuffle scan, offset search, component votes) is stated here as plain loops; `votes` chooses how the need_* flags are formed:
// 0 = every component always, 1 = exactly what the block's position uses (the two extremes the warp vote lies between).
#include "shim/cuda_runtime.h"
#include "h264_mc_block.cuh"
#include "../../include/avdsp_b200.h"
// the register-resident residual kernel (one lane per block, lanes never communicate): compiled unchanged, a launch = its body once per thread
#include "../../libav_b200/csrc/h264_residual.cu"

extern "C" int hostsim_h264_residual(const FFH264ResidualMB *mbs, size_t n, int16_t *coeffs, size_t coeff_stride, const uint8_t *nnzc,
                                     uint8_t *luma, uint8_t *cb, uint8_t *cr, int ls, int uvls)
{ return avb::launch_h264_residual_v2(mbs, n, coeffs, coeff_stride, nnzc, luma, cb, cr, ls, uvls, nullptr); }

extern "C" int hostsim_h264_mc(const FFH264MCRecord *recs, size_t n, const FFH264RefPlanes *refs, uint8_t *dy, uint8_t *dcb, uint8_t *dcr,
                               int ls, int uvls, int pw, int ph, int votes)
{
    for (int pass = 0; pass < 2; pass++)
        for (size_t i = 0; i < n; i++) {
            const FFH264MCRecord &r = recs[i];
            if ((r.avg != 0) != (pass != 0)) continue;
            const int ly0 = (r.y / ph) * ph;
            const FFH264RefPlanes &rp = refs[r.ref];
            avb::McPlanes pl = { rp.y, rp.cb, rp.cr };
            const bool aligned = !(((uintptr_t)rp.y | (uintptr_t)rp.cb | (uintptr_t)rp.cr | (uintptr_t)ls | (uintptr_t)uvls) & 3);
            for (int by = 0; by < r.h / 4; by++)
                for (int bx = 0; bx < r.w / 4; bx++) {
                    const int x = r.x + 4 * bx, y = r.y + 4 * by, mx = r.mvx + 4 * x, my = r.mvy + 4 * y, fx = mx & 3, fy = my & 3;
                    const bool uj = (fx == 2 && fy != 0) || (fy == 2 && fx != 0), uh = fx != 0 && fy != 2, uv = fy != 0 && fx != 2;
                    if (avb::mc_block_inside(pw, ph, ly0, mx, my, aligned))
                        avb::mc_block<false>(pl, dy, dcb, dcr, ls, uvls, pw, ph, ly0, x, y, mx, my, r.avg, votes ? uh : true, votes ? uv : true, votes ? uj : true);
                    else
                        avb::mc_block<true>(pl, dy, dcb, dcr, ls, uvls, pw, ph, ly0, x, y, mx, my, r.avg, votes ? uh : true, votes ? uv : true, votes ? uj : true);
                }
        }
    return 0;
}
