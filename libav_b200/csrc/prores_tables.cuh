// libav_b200/csrc/prores_tables.cuh -- the ProRes scan tables and codebooks (libavcodec/proresdata.c, restated), one copy for the encoder
// (prores_enc.cuh) and the decoder (prores_dec.cuh).  Constant memory on the device; plain arrays in the host build (tests/hostsim/).
#pragma once
#include "common.cuh"

namespace avb {

#ifdef AVB_HOSTSIM
#define PE_TABLE static const
#else
#define PE_TABLE static __constant__ const
#endif

// libavcodec/proresdata.c, restated
PE_TABLE uint8_t pe_scan[2][64] = {
    {  0,  1,  8,  9,  2,  3, 10, 11, 16, 17, 24, 25, 18, 19, 26, 27,  4,  5, 12, 20, 13,  6,  7, 14, 21, 28, 29, 22, 15, 23, 30, 31,
      32, 33, 40, 48, 41, 34, 35, 42, 49, 56, 57, 50, 43, 36, 37, 44, 51, 58, 59, 52, 45, 38, 39, 46, 53, 60, 61, 54, 47, 55, 62, 63 },
    {  0,  8,  1,  9, 16, 24, 17, 25,  2, 10,  3, 11, 18, 26, 19, 27, 32, 40, 33, 34, 41, 48, 56, 49, 42, 35, 43, 50, 57, 58, 51, 59,
       4, 12,  5,  6, 13, 20, 28, 21, 14,  7, 15, 22, 29, 36, 44, 37, 30, 23, 31, 38, 45, 52, 60, 53, 46, 39, 47, 54, 61, 62, 55, 63 },
};
PE_TABLE uint8_t pe_dc_codebook[4] = { 0x04, 0x28, 0x4D, 0x70 };
PE_TABLE uint8_t pe_ac_codebook[7] = { 0x04, 0x28, 0x4C, 0x05, 0x29, 0x06, 0x0A };
PE_TABLE uint8_t pe_run_to_cb[16] = { 5, 5, 3, 3, 0, 4, 4, 4, 4, 1, 1, 1, 1, 1, 1, 2 };
PE_TABLE uint8_t pe_lev_to_cb[10] = { 0, 6, 3, 5, 0, 1, 1, 1, 1, 2 };
constexpr int PE_FIRST_DC_CB = 0xB8;

}  // namespace avb
