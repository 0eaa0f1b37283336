// libav_b200/csrc/sws_fused.h -- what the two same-size yuv420p -> rgb24 / bgr24 kernels share: the launch arguments, the per-row-pair
// tables the host builds from the vertical chroma bank, and the packed clip of the output stage.
//   swscale.cu        sws_fused_rgb24_kernel (any pitch, byte tails), sws_fused_rgb24_v3_kernel (LDG, 8-byte aligned pitches)
//   sws_fused_tma.cu  sws_fused_rgb24_tma_kernel (the 4K benchmark path: TMA-staged line buffers, persistent warps)
#pragma once
#include "common.cuh"
#include "sws_filter.h"

namespace avb {

struct FusedArgs {
    const uint8_t *y, *u, *v; uint8_t *dst;
    int yStride, uStride, vStride, dstStride;
    size_t yFrame, uFrame, vFrame, dstFrame;      // byte distance between consecutive frames of a batch
    int rp0 = 0, rp1 = 0x7fffffff;                 // row-pair range of this launch (bands of the host pipeline)
};

// Per row pair, for the TMA kernel.  The two rows of pair rp are output lines 2 rp and 2 rp + 1; row r filters the four chroma lines
// first_r .. first_r + 3 (clamped into the plane: swscale.c:463, :592-616) with taps (k01_r & 0xffff, k01_r >> 16, k23_r & 0xffff, k23_r >> 16)
// -- the int16 pairs dp2a takes.  A warp's tile is four consecutive pairs (rp & ~3 .. | 3): `base` is the first chroma line its TMA box
// starts at, `interior` says that pair q of the tile starts at base + q, its second row one line lower, and no line needs clamping.
struct SwsPairTapsT {
    uint32_t k01_0, k23_0, k01_1, k23_1;
    int first0, first1;
    int base, interior;
};

// four 32-bit sums -> one word of clip_u8(sum >> 16): the upper half-words of two sums are gathered by one PRMT, clipped
// two at a time (packed s16 min + relu) and the four low bytes gathered by a third PRMT: 5 ALU-pipe instructions instead
// of 4 shifts + 2 saturating packs.  Valid because |sum >> 16| < 2^15.
__device__ __forceinline__ uint32_t pack4_hi16_sat(int w0, int w1, int w2, int w3)
{
    const uint32_t h01 = __byte_perm((uint32_t)w0, (uint32_t)w1, 0x7632), h23 = __byte_perm((uint32_t)w2, (uint32_t)w3, 0x7632);
    const uint32_t c01 = __vimin_s16x2_relu(h01, 0x00FF00FFu), c23 = __vimin_s16x2_relu(h23, 0x00FF00FFu);
    return __byte_perm(c01, c23, 0x6420);
}
__device__ __forceinline__ int sat255(int v) { return __vimin_s32_relu(v, 255); }       // max(min(v, 255), 0), one VIMNMX

#ifndef AVB_HOSTSIM
// 0 launched, -1 error (sticky message set), 1 not applicable (pitches / pointers the tensor maps cannot describe): the caller runs
// the LDG kernel instead.  `taps` is the device copy of SwsPairTapsT[dstH / 2].  `tickets` is the kernel's tile counter: one int,
// zero before the first launch, which every launch leaves at zero; launches that share it must be ordered on one stream.
int sws_fused_tma_launch(const RgbConstants &k, int bgr, int dstW, int dstH, int chrSrcW, int chrSrcH, const FusedArgs &a,
                         const SwsPairTapsT *taps, int *tickets, int nframes, cudaStream_t st);
#endif

}  // namespace avb
