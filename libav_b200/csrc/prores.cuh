// libav_b200/csrc/prores.cuh -- the ProRes picture reconstruction of prores.cu (dequantisation, IDCT and store of a picture's staged
// coefficient blocks) as the whole-packet decoder (prores_dec.cu) launches it.
#pragma once
#include "common.cuh"
#include "../../include/avdsp_b200.h"

namespace avb {

// decode_picture's slice grid: 1 << swf macroblocks per slice, the width halving at the right edge until the slice fits
__host__ __device__ inline int pr_slices_per_row(int mb_w, int swf)
{
    const int rem = mb_w & ((1 << swf) - 1);
    return (mb_w >> swf) + (rem & 1) + ((rem >> 1) & 1) + ((rem >> 2) & 1);
}

// A slice's plane status: byte p (0 Y, 1 U, 2 V) is 1 when that plane's coefficients decoded.  decode_slice returns at its first failing
// plane, so plane p is written only when planes 0..p all decoded.
__host__ __device__ __forceinline__ bool pr_plane_written(uint32_t status, int p)
{
    const uint32_t need = 0x00010101u & ((0x100u << (8 * p)) - 1);
    return (status & need) == need;
}

// ff_prores_decode_pictures_cuda's launches for pictures it has checked.  status: NULL (every slice writes every plane), or per picture a
// device array of its slices' plane status words.
int launch_prores_pictures(const FFProresPictureWork *pictures, int n, cudaStream_t st, const uint32_t *const *status = nullptr);

}  // namespace avb
