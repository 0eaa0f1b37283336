// libav_b200/csrc/mpv_quant.cuh -- the encoder's plain quantiser, ff_dct_quantize_c (libavcodec/mpegvideo_enc.c:4371-4450) after its
// forward DCT and noise reduction, on one thread's int16 block.  Shared by the quant_psnr / bit / rd metrics (me_cmp_enc.cu) and the
// batched quantiser (mpv_quant.cu).  Thread-local arithmetic only (also compiled by tests/hostsim/).
#pragma once
#include "common.cuh"
#include "../../include/avdsp_b200.h"

namespace avb {

constexpr int MPV_QMAT_SHIFT = 22, MPV_QUANT_BIAS_SHIFT = 8;      // QMAT_SHIFT, QUANT_BIAS_SHIFT (mpegvideo_enc.c:65-68)

// The intra DC division by dc_q (= (h263_aic ? 1 : dc_scale) << 3) with C's truncating '/', then the biased threshold quantiser in scan
// order from start_i (1 intra, 0 inter).  bias is intra_quant_bias / inter_quant_bias in QUANT_BIAS_SHIFT units.  The C code's two loops
// (find the last kept position from the back, then quantise up to it) reduce to "kept or zero" per position plus the largest kept position.
// Returns last_non_zero; max = the OR of the kept magnitudes (overflow = max_qcoeff < max).  The product block[j] * qmat[j] wraps at 32 bits
// like gcc's code for the reference.
__device__ __forceinline__ int mpv_quantize(int16_t *t, bool intra, int dc_q, const int32_t *qmat, int bias, const uint8_t *scantable, int &max)
{
    bias *= 1 << (MPV_QMAT_SHIFT - MPV_QUANT_BIAS_SHIFT);
    const unsigned t1 = (1u << MPV_QMAT_SHIFT) - (unsigned)bias - 1u, t2 = t1 << 1;
    int last = intra ? 0 : -1;
    max = 0;
    if (intra) t[0] = (int16_t)((t[0] + (dc_q >> 1)) / dc_q);
    for (int i = intra ? 1 : 0; i < 64; i++) {
        const int j = scantable[i];
        const int level = (int)((unsigned)(int)t[j] * (unsigned)qmat[j]);
        if ((unsigned)level + t1 > t2) {
            const int m = level > 0 ? (int)((unsigned)bias + (unsigned)level) >> MPV_QMAT_SHIFT : (int)((unsigned)bias - (unsigned)level) >> MPV_QMAT_SHIFT;
            t[j] = (int16_t)(level > 0 ? m : -m);
            max |= m;
            last = i;
        } else t[j] = 0;
    }
    return last;
}

// device copy of a codec's VLC length tables (intra len, intra last, inter len, inter last at 8192-byte steps, then the 512-byte luma DC
// table), cached by host address and checked against a checksum when verify is set (me_cmp_enc.cu)
const uint8_t *vlc_device(const FFMECmpVlcTables *v, const char *where, bool verify = false);

}  // namespace avb
