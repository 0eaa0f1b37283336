// libav_b200/csrc/idctdsp.cu -- batched 8x8 "simple" IDCT family + clamped pixel ops + block clear
// for sm_90a.  Replaces, bit-exactly, the C slots of IDCTDSPContext / BlockDSPContext:
//   ff_simple_idct_put_8 / _add_8 / ff_simple_idct_8   libavcodec/simple_idct_template.c:289-326
//   put/put_signed/add_pixels_clamped_c                libavcodec/idctdsp.c:85-145
//   clear_block(s)                                     libavcodec/blockdsp.c:29-37
//
// Work mapping: ONE THREAD PER 8x8 BLOCK, 32 blocks (4 KB of coefficients) per warp.
//   * the warp's 4 KB is brought in with 8 fully coalesced 512-byte cp.async (LDGSTS) requests into
//     a 128-byte-row XOR-swizzled shared tile (chunk c of block b lands at chunk c ^ (b & 7)), so
//     the per-thread row reads (LDS.128, thread = block) are bank-conflict free;
//   * both passes run in registers: no shuffles, no second transpose.  Integer semantics follow
//     the reference exactly: W4 = 16383, the DC-only row shortcut (x0 << 3), int16 truncation of the
//     row pass, rounding folded in the column DC term, 32-bit wrap-around arithmetic;
//   * results leave as one 8-byte row store per (thread,row): with raster-ordered blocks a warp
//     writes 256 contiguous bytes per picture row.
// Two tiles per warp are double-buffered so the next group's loads fly during the math.
// Algorithmic traffic: put 128 B in + 64 B out (+4 B offset) per block; add 256 B; idct 256 B.
// The two passes are a policy of the kernel template (SimpleIdct here, XvidIdct in xvid_idct.cuh for ff_xvid_idct): everything else
// -- staging, fetch, addressing, fused clear and dequantisation -- is shared.  The FAAN IDCT (float between the passes) has a kernel body of
// its own, faan_idct_kernel, over the same staging and inverse quantisers.
#include "common.cuh"
#include <type_traits>
#include <cuda.h>            // CUtensorMap only; the encoder is looked up at run time (no libcuda link dependency)
#include "idct_dq.h"
#include "xvid_idct.cuh"
#include "faan_dct.cuh"
#include "block_stage.cuh"

namespace avb {

enum { C1 = 22725, C2 = 21407, C3 = 19266, C4 = 16383, C5 = 12873, C6 = 8867, C7 = 4520 };

// Shared butterflies.  K = 1 for the column pass, 32 for the row pass: the row pass needs bits [26:11] of each sum
// (the int16 the reference stores back), and with every constant pre-multiplied by 32 those bits land in the upper
// half-word of the 32-bit wrap-around result, ready for a byte-permute -- no shift per output.  Multiplying all terms
// by 32 commutes with the mod-2^32 arithmetic, so the selected bits are identical.
// s[k] = e[k] + o[k] is accumulated as one IMAD chain that starts from e[k]; d[k] = e[k] - o[k] = 2 e[k] - s[k] then
// costs a single 3-input add.
template <int K>
__device__ __forceinline__ void butterfly(int base, int x1, int x2, int x3, int x4, int x5, int x6, int x7,
                                          int (&s)[4], int (&d)[4])
{
    const int b0 = base + (K * C4) * x4, b1 = base - (K * C4) * x4;
    const int p  = (K * C2) * x2 + (K * C6) * x6;
    const int q  = (K * C6) * x2 - (K * C2) * x6;
    const int e0 = b0 + p, e3 = b0 - p, e1 = b1 + q, e2 = b1 - q;
    s[0] = e0 + (K * C1) * x1 + (K * C3) * x3 + (K * C5) * x5 + (K * C7) * x7;
    s[1] = e1 + (K * C3) * x1 - (K * C7) * x3 - (K * C1) * x5 - (K * C5) * x7;
    s[2] = e2 + (K * C5) * x1 - (K * C1) * x3 + (K * C7) * x5 + (K * C3) * x7;
    s[3] = e3 + (K * C7) * x1 - (K * C5) * x3 + (K * C3) * x5 - (K * C1) * x7;
    d[0] = e0 + e0 - s[0];
    d[1] = e1 + e1 - s[1];
    d[2] = e2 + e2 - s[2];
    d[3] = e3 + e3 - s[3];
}

template <bool MH> __device__ __forceinline__ int hi16x(uint32_t w) { return sra<16, MH>((int)w); }

// Row pass on one packed row (4 words = 8 int16); result is the int16-truncated row, packed.
template <bool MH>
__device__ __forceinline__ uint4 row_pass(uint4 r)
{
    int x0 = lo16s(r.x), x1 = hi16x<MH>(r.x), x2 = lo16s(r.y), x3 = hi16x<MH>(r.y);
    int x4 = lo16s(r.z), x5 = hi16x<MH>(r.z), x6 = lo16s(r.w), x7 = hi16x<MH>(r.w);
    // all seven AC terms zero -> every output is (x0 << 3): feed base = (x0 << 14) * 32 through the same datapath
    // (the butterflies add zero), simple_idct_template.c:94-106
    bool dc_only = ((r.x & 0xffff0000u) | r.y | r.z | r.w) == 0;
    int base = dc_only ? (x0 << 19) : ((32 * C4) * x0 + (1 << 15));
    int s[4], d[4];
    butterfly<32>(base, x1, x2, x3, x4, x5, x6, x7, s, d);
    uint4 o;                                   // upper half-words = (int16_t)(sum >> 11)
    o.x = __byte_perm((uint32_t)s[0], (uint32_t)s[1], 0x7632);
    o.y = __byte_perm((uint32_t)s[2], (uint32_t)s[3], 0x7632);
    o.z = __byte_perm((uint32_t)d[3], (uint32_t)d[2], 0x7632);
    o.w = __byte_perm((uint32_t)d[1], (uint32_t)d[0], 0x7632);
    return o;
}

// Column pass for column x given the eight row words that contain it; out[y] = value >> 20.
template <int HI, bool MH>
__device__ __forceinline__ void col_pass(const uint32_t (&w)[8], int (&out)[8])
{
    int x[8];
#pragma unroll
    for (int k = 0; k < 8; k++) x[k] = HI ? hi16x<MH>(w[k]) : lo16s(w[k]);
    int base = C4 * (x[0] + 32);            // (1 << 19) / 16383 == 32
    int s[4], d[4];
    butterfly<1>(base, x[1], x[2], x[3], x[4], x[5], x[6], x[7], s, d);
#pragma unroll
    for (int k = 0; k < 4; k++) { out[k] = sra<20, MH>(s[k]); out[7 - k] = sra<20, MH>(d[k]); }
}

// the transform policy of simple_idct_kernel: this file's simple IDCT (xvid_idct.cuh has the Xvid one)
struct SimpleIdct {
    template <bool MH> static __device__ __forceinline__ uint4 row(uint4 v, int) { return row_pass<MH>(v); }
    template <int HI, bool MH> static __device__ __forceinline__ void col(const uint32_t (&w)[8], int (&out)[8]) { col_pass<HI, MH>(w, out); }
};

__device__ __forceinline__ size_t block_dst(const uint32_t *__restrict__ dst_off, size_t i,
                                            int tiles_per_row, ptrdiff_t stride)
{
    if (dst_off) return dst_off[i];
    size_t ty = i / (unsigned)tiles_per_row, tx = i - ty * (unsigned)tiles_per_row;
    return ty * 8 * (size_t)stride + tx * 8;
}

constexpr int IDCT_WARPS = 4;   // warps per CTA; each owns 2 x 4 KB of shared memory

// MODE 0: put, 1: add, 2: plain (in place int16).  CLEAR: also zero the coefficient block
// afterwards (fused BlockDSPContext.clear_block, what every caller does next).
// cp.async / ld.shared on raw 32-bit shared addresses: every per-lane offset below is loop invariant, so the steady
// state of the loop issues no address arithmetic beyond one add per buffer flip.
__device__ __forceinline__ void cp_async16_s(unsigned saddr, const void *gmem)
{ asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" :: "r"(saddr), "l"(gmem) : "memory"); }
__device__ __forceinline__ void cp_async16_sz(unsigned saddr, const void *gmem, int bytes)
{ asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" :: "r"(saddr), "l"(gmem), "r"(bytes) : "memory"); }
__device__ __forceinline__ uint4 lds128(unsigned saddr)
{
    uint4 r;
    asm volatile("ld.shared.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w) : "r"(saddr));
    return r;
}

// ---------------------------------------------------------------------------------------------------
// Inverse quantisation in front of the IDCT: MpegEncContext.dct_unquantize_* (libavcodec/mpegvideo.c:51-270) as a
// per-coefficient rule.  DQ: 0 none, 1 + kind otherwise (kind 0 mpeg1_intra 1 mpeg1_inter 2 mpeg2_intra 3 mpeg2_intra
// bitexact 4 mpeg2_inter 5 h263_intra 6 h263_inter).  One thread owns one block, so the raster index j is the same in
// every lane at every unrolled step: matrix[j] and rank[j] are kernel-parameter (constant bank) operands.
// ---------------------------------------------------------------------------------------------------
struct DqLane { int qscale, limit, dc_scale, qadd; };

template <int KIND>
__device__ __forceinline__ DqLane dq_lane(uint32_t rec, const DqTables &T)
{
    DqLane L;
    L.qscale = rec & 255;
    const int last = (int)(int8_t)(rec >> 8), ac_pred = (rec >> 24) & 1;
    L.dc_scale = (rec >> 16) & 255;
    if (KIND >= 5) L.limit = (KIND == 5 && ac_pred) ? 63 : (last < 0 ? -1 : (int)T.raster_end[last]);
    else           L.limit = ((KIND == 2 || KIND == 3 || KIND == 4) && T.alternate_scan) ? 63 : last;
    L.qadd = (KIND == 5 && T.h263_aic) ? 0 : (L.qscale - 1) | 1;
    return L;
}

// Sign-free forms of the C code's "negate, scale, negate back": with p = level * (qscale * matrix) the magnitude shift is
// a division that truncates towards zero, u = (p + ((p >> 31) & (2^k - 1))) >> k; MPEG-1's oddification (v - 1) | 1 of
// the magnitude is (u - 1 - s) | 1 with s = level >> 31.  Exact while |level| * qscale * matrix < 2^31, which holds for
// every int16 level with qscale <= 112 and 8-bit matrices (what the bitstreams can carry); include/avdsp_b200.h says so.
template <int KIND>
__device__ __forceinline__ int dq_coef(int level, int j, const DqTables &T, const DqLane &L, int &sum)
{
    constexpr bool INTRA = KIND == 0 || KIND == 2 || KIND == 3 || KIND == 5;
    if (INTRA && j == 0) return (KIND == 5 && T.h263_aic) ? level : level * L.dc_scale;
    const int pos = KIND >= 5 ? j : (int)T.rank[j];
    const int s = level >> 31;
    int v;
    if (KIND == 0 || KIND == 2 || KIND == 3) {
        const int p = level * (L.qscale * (int)T.intra[j]);
        v = (p + ((p >> 31) & 7)) >> 3;
        if (KIND == 0) v = (v - 1 - s) | 1;
    } else if (KIND == 1 || KIND == 4) {
        const int p = (2 * level + 1 + 2 * s) * (L.qscale * (int)T.inter[j]);
        v = (p + ((p >> 31) & 15)) >> 4;
        if (KIND == 1) v = (v - 1 - s) | 1;
    } else {
        v = level * (2 * L.qscale) + ((L.qadd ^ s) - s);
    }
    // a zero level stays zero by itself under the MPEG-2 intra rule; everywhere else it must be kept out explicitly
    const bool coded = (KIND == 2 || KIND == 3) ? pos <= L.limit : (pos <= L.limit && level != 0);
    if (KIND == 3 || KIND == 4) sum += coded ? v : 0;
    return coded ? v : level;
}

// one row (8 packed int16) of a block; results are stored back as int16 exactly like the C code's block[j] = level
template <int KIND>
__device__ __forceinline__ uint4 dq_row(uint4 w, int r, const DqTables &T, const DqLane &L, int &sum)
{
    const uint32_t in[4] = { w.x, w.y, w.z, w.w };
    uint32_t out[4];
#pragma unroll
    for (int c = 0; c < 4; c++)
        out[c] = pack16(dq_coef<KIND>(lo16s(in[c]), 8 * r + 2 * c, T, L, sum), dq_coef<KIND>(hi16s(in[c]), 8 * r + 2 * c + 1, T, L, sum));
    if ((KIND == 3 || KIND == 4) && r == 7) out[3] ^= (uint32_t)(sum & 1) << 16;       // mismatch control on block[63]
    return make_uint4(out[0], out[1], out[2], out[3]);
}

// MODE 0: put, 1: add, 2: plain (in place int16).  CLEAR: also zero the coefficient block
// afterwards (fused BlockDSPContext.clear_block, what every caller does next).
// DQ != 0: dequantise (kind DQ - 1) in front of the row pass -- put_dct / add_dequant_dct of libavcodec/mpegvideo.c:1401-1427
// in one kernel; an `add` block with block_last_index < 0 is skipped like the C code skips it.
struct DqArgs { const uint32_t *recs; DqTables t; };
struct NoDq {};
struct NoTma {};
// TMA: the warp's 4 KB group arrives by ONE cp.async.bulk.tensor issued by lane 0 (2-D tensor map over the block array,
// box 32 blocks x 128 B, SWIZZLE_128B = the same chunk ^ (block & 7) layout the cp.async path builds by hand) and is
// awaited on an mbarrier, instead of eight cp.async per lane.
// XF: the transform (SimpleIdct, XvidIdct): its row pass on each packed row and its column pass; everything else is shared.
template <int MODE, bool CLEAR, int MINB = 5, bool MH = false, int DQ = 0, bool TMA = false, class XF = SimpleIdct>
__global__ void __launch_bounds__(IDCT_WARPS * 32, MINB)
simple_idct_kernel(int16_t *__restrict__ blocks, uint8_t *__restrict__ frame,
                   const uint32_t *__restrict__ dst_off, ptrdiff_t stride, size_t n, int tiles_per_row,
                   const typename std::conditional<DQ != 0, DqArgs, NoDq>::type dq = {},
                   const __grid_constant__ typename std::conditional<TMA, CUtensorMap, NoTma>::type tmap = {})
{
    __shared__ __align__(1024) uint4 tile[IDCT_WARPS][2][256];  // 32 blocks x 8 chunks of 16 B (1 KB alignment: TMA swizzle atom)
    __shared__ __align__(8) uint64_t mbar[IDCT_WARPS][2];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const size_t groups = (n + 31) / 32;
    const size_t gstride = (size_t)gridDim.x * IDCT_WARPS;
    size_t g = (size_t)blockIdx.x * IDCT_WARPS + warp;

    // loop-invariant shared-memory byte offsets.  A 512-byte slab j of the group holds blocks 4j..4j+3; lane writes chunk
    // c = lane & 7 of block 4j + (lane >> 3) to chunk position c ^ (block & 7), and (block & 7) = 4 (j & 1) + (lane >> 3).
    const unsigned tile_s = (unsigned)__cvta_generic_to_shared(&tile[warp][0][0]);
    const int l3 = lane >> 3, lc = lane & 7;
    const unsigned wr_even = (unsigned)(l3 * 8 + (lc ^ l3)) * 16, wr_odd = (unsigned)(l3 * 8 + (lc ^ (4 + l3))) * 16;
    const unsigned rd_base = (unsigned)lane * 128, rd_key = (unsigned)lc << 4;

    const unsigned mbar_s = (unsigned)__cvta_generic_to_shared(&mbar[warp][0]);
    if constexpr (TMA) {
        if (lane == 0) {
            asm volatile("mbarrier.init.shared::cta.b64 [%0], 1;" :: "r"(mbar_s) : "memory");
            asm volatile("mbarrier.init.shared::cta.b64 [%0], 1;" :: "r"(mbar_s + 8) : "memory");
            asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
        }
        __syncwarp();
    }
    auto issue = [&](size_t grp, unsigned tb) {
        if constexpr (TMA) {
            if (lane == 0) {
                const unsigned mb = mbar_s + ((tb - tile_s) >> 9);                 // buffer 0 -> +0, buffer 1 (4096) -> +8
                asm volatile("fence.proxy.async.shared::cta;" ::: "memory");     // the buffer was last touched by ordinary loads
                asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" :: "r"(mb), "r"(4096) : "memory");
                asm volatile("cp.async.bulk.tensor.2d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3}], [%4];"
                             :: "r"(tb), "l"(reinterpret_cast<uint64_t>(&tmap)), "r"(0), "r"((int)(grp * 32)), "r"(mb) : "memory");
            }
            return;
        }
        const char *src = reinterpret_cast<const char *>(blocks) + grp * 4096 + lane * 16;
        if (grp * 32 + 32 <= n) {
#pragma unroll
            for (int j = 0; j < 8; j++) cp_async16_s(tb + j * 512 + ((j & 1) ? wr_odd : wr_even), src + j * 512);
        } else {                                              // ragged last group: zero-fill the missing blocks
#pragma unroll
            for (int j = 0; j < 8; j++) {
                const bool ok = grp * 32 + j * 4 + l3 < n;
                cp_async16_sz(tb + j * 512 + ((j & 1) ? wr_odd : wr_even), ok ? src + j * 512 : reinterpret_cast<const char *>(blocks), ok ? 16 : 0);
            }
        }
        cp_async_commit();
    };

    // raster-of-tiles destination: (ty, tx) of this lane's block advances by a constant step per iteration (no division)
    size_t ty = 0; unsigned tx = 0, step_q = 0, step_r = 0;
    if (MODE != 2 && !dst_off) {
        const size_t i0 = g * 32 + lane, st = gstride * 32;
        ty = i0 / (unsigned)tiles_per_row; tx = (unsigned)(i0 - ty * (unsigned)tiles_per_row);
        step_q = (unsigned)(st / (unsigned)tiles_per_row); step_r = (unsigned)(st - (size_t)step_q * (unsigned)tiles_per_row);
    }

    unsigned buf = 0, uses = 0;
    if (g < groups) issue(g, tile_s);
    for (; g < groups; g += gstride, buf ^= 4096u, uses++) {
        const size_t gn = g + gstride;
        const unsigned tb = tile_s + buf;
        if constexpr (TMA) {
            if (gn < groups) issue(gn, tile_s + (buf ^ 4096u));
            const unsigned mb = mbar_s + (buf >> 9), parity = (uses >> 1) & 1;      // k-th use of a buffer completes phase k
            asm volatile("{\n.reg .pred p;\nIDCT_TMA_WAIT_%=:\nmbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n@p bra IDCT_TMA_DONE_%=;\nbra IDCT_TMA_WAIT_%=;\nIDCT_TMA_DONE_%=:\n}"
                         :: "r"(mb), "r"(parity) : "memory");
        } else {
            if (gn < groups) { issue(gn, tile_s + (buf ^ 4096u)); cp_async_wait<1>(); } else cp_async_wait<0>();
        }
        __syncwarp();

        const size_t i = g * 32 + lane;
        bool live = i < n;
        uint4 row[8];
        if constexpr (DQ != 0) {
            const uint32_t rec = live ? dq.recs[i] : 0;
            const DqLane L = dq_lane<DQ - 1>(rec, dq.t);
            if (MODE == 1 && (int8_t)(rec >> 8) < 0) live = false;
            int sum = -1;
#pragma unroll
            for (int r = 0; r < 8; r++)
                row[r] = XF::template row<MH>(dq_row<DQ - 1>(lds128(tb + rd_base + (((unsigned)r << 4) ^ rd_key)), r, dq.t, L, sum), r);
        } else {
#pragma unroll
            for (int r = 0; r < 8; r++) row[r] = XF::template row<MH>(lds128(tb + rd_base + (((unsigned)r << 4) ^ rd_key)), r);
        }
        __syncwarp();     // this buffer is free for the load issued two iterations from now

        if (MODE == 2) {
            // plain idct: results go back in place as int16, column by column pair
            uint32_t o[8][4];
#pragma unroll
            for (int c = 0; c < 4; c++) {
                uint32_t w[8];
#pragma unroll
                for (int r = 0; r < 8; r++) w[r] = c == 0 ? row[r].x : c == 1 ? row[r].y : c == 2 ? row[r].z : row[r].w;
                int lo[8], hi[8];
                XF::template col<0, MH>(w, lo);
                XF::template col<1, MH>(w, hi);
#pragma unroll
                for (int y = 0; y < 8; y++) o[y][c] = pack16(lo[y], hi[y]);
            }
            if (live) {
                uint4 *dst = reinterpret_cast<uint4 *>(blocks) + i * 8;
#pragma unroll
                for (int y = 0; y < 8; y++) dst[y] = make_uint4(o[y][0], o[y][1], o[y][2], o[y][3]);
            }
        } else {
            uint8_t *dst = frame;
            if (dst_off) dst += live ? dst_off[i] : 0;
            else {
                dst += ty * 8 * (size_t)stride + (size_t)tx * 8;
                tx += step_r; ty += step_q;
                if (tx >= (unsigned)tiles_per_row) { tx -= (unsigned)tiles_per_row; ty++; }
            }
            uint2 px[8];
            if (MODE == 1 && live) {
#pragma unroll
                for (int y = 0; y < 8; y++) px[y] = *reinterpret_cast<const uint2 *>(dst + y * stride);
            }
            uint32_t o[8][2];
#pragma unroll
            for (int h = 0; h < 2; h++) {
                int v[4][8];
#pragma unroll
                for (int c = 0; c < 2; c++) {
                    uint32_t w[8];
#pragma unroll
                    for (int r = 0; r < 8; r++)
                        w[r] = h == 0 ? (c == 0 ? row[r].x : row[r].y) : (c == 0 ? row[r].z : row[r].w);
                    XF::template col<0, MH>(w, v[2 * c]);
                    XF::template col<1, MH>(w, v[2 * c + 1]);
                }
#pragma unroll
                for (int y = 0; y < 8; y++) {
                    if (MODE == 1) {
                        uint32_t p = h == 0 ? px[y].x : px[y].y;
                        o[y][h] = pack4_sat_u8(v[0][y] + byte_of(p, 0), v[1][y] + byte_of(p, 1),
                                               v[2][y] + byte_of(p, 2), v[3][y] + byte_of(p, 3));
                    } else {
                        o[y][h] = pack4_sat_u8(v[0][y], v[1][y], v[2][y], v[3][y]);
                    }
                }
            }
            if (live) {
#pragma unroll
                for (int y = 0; y < 8; y++)
                    *reinterpret_cast<uint2 *>(dst + y * stride) = make_uint2(o[y][0], o[y][1]);
            }
            if (CLEAR && live) {
                uint4 *b = reinterpret_cast<uint4 *>(blocks) + i * 8;
#pragma unroll
                for (int y = 0; y < 8; y++) b[y] = make_uint4(0, 0, 0, 0);
            }
        }
    }
}

// The FAAN IDCT (ff_faanidct / _put / _add, faan_dct.cuh) over the same staging: its data between the passes is float, so it has its own
// body rather than a transform policy of simple_idct_kernel.  One thread per block; the lane's eight rows arrive as LDS.128 from the
// warp's swizzled tile (WarpBlockStage), both passes run in registers.  MODE 0 put, 1 add, 2 in place (the result goes back through the
// tile and leaves as coalesced 512-byte stores); CLEAR zeroes a put / add block afterwards; DQ != 0 fuses inverse quantiser kind DQ - 1
// in front, with the skipping rule of simple_idct_kernel.  put / add leave the coefficients untouched, as the C functions do.
template <int MODE, bool CLEAR, int DQ = 0>
__global__ void __launch_bounds__(IDCT_WARPS * 32)
faan_idct_kernel(int16_t *__restrict__ blocks, uint8_t *__restrict__ frame, const uint32_t *__restrict__ dst_off, ptrdiff_t stride, size_t n,
                 int tiles_per_row, const typename std::conditional<DQ != 0, DqArgs, NoDq>::type dq = {})
{
    __shared__ __align__(128) uint4 tile[IDCT_WARPS][2][256];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const WarpBlockStage S(&tile[warp][0][0], lane);
    const size_t groups = (n + 31) / 32, gstride = (size_t)gridDim.x * IDCT_WARPS;
    size_t g = (size_t)blockIdx.x * IDCT_WARPS + warp;
    unsigned buf = 0;
    if (g < groups) S.issue(blocks, g, n, S.buffer(0));
    for (; g < groups; g += gstride, buf ^= 4096u) {
        const size_t gn = g + gstride;
        const unsigned tb = S.buffer(buf);
        if (gn < groups) { S.issue(blocks, gn, n, S.buffer(buf ^ 4096u)); cp_async_wait<1>(); } else cp_async_wait<0>();
        __syncwarp();
        const size_t i = g * 32 + lane;
        bool live = i < n;
        float t[8][8];
        [[maybe_unused]] uint32_t rec = 0;
        [[maybe_unused]] DqLane L = {};
        [[maybe_unused]] int sum = -1;
        if constexpr (DQ != 0) {
            rec = live ? dq.recs[i] : 0;
            L = dq_lane<DQ - 1>(rec, dq.t);
            if (MODE == 1 && (int8_t)(rec >> 8) < 0) live = false;
        }
#pragma unroll
        for (int r = 0; r < 8; r++) {
            uint4 w = S.row(tb, r);
            if constexpr (DQ != 0) w = dq_row<DQ - 1>(w, r, dq.t, L, sum);
            const int x[8] = { lo16s(w.x), hi16s(w.x), lo16s(w.y), hi16s(w.y), lo16s(w.z), hi16s(w.z), lo16s(w.w), hi16s(w.w) };
            faan::idct_row(x, r, t[r]);
        }
#pragma unroll
        for (int c = 0; c < 8; c++) {
            float col[8];
#pragma unroll
            for (int k = 0; k < 8; k++) col[k] = t[k][c];
            faan::idct_1d(col);
#pragma unroll
            for (int k = 0; k < 8; k++) t[k][c] = col[k];
        }
        if (MODE == 2) {
            __syncwarp();                                    // every lane has read its rows: the tile takes the results
#pragma unroll
            for (int y = 0; y < 8; y++) {
                int v[8];
#pragma unroll
                for (int c = 0; c < 8; c++) v[c] = __float2int_rn(t[y][c]);
                S.put_row(tb, y, make_uint4(pack16(v[0], v[1]), pack16(v[2], v[3]), pack16(v[4], v[5]), pack16(v[6], v[7])));
            }
            S.flush(blocks, g, n, tb);
        } else if (live) {
            uint8_t *dst = frame + block_dst(dst_off, i, tiles_per_row, stride);
#pragma unroll
            for (int y = 0; y < 8; y++) {
                int v[8];
#pragma unroll
                for (int c = 0; c < 8; c++) v[c] = __float2int_rn(t[y][c]);
                if (MODE == 1) {
                    const uint2 p = *reinterpret_cast<const uint2 *>(dst + y * stride);
#pragma unroll
                    for (int k = 0; k < 4; k++) { v[k] += byte_of(p.x, k); v[4 + k] += byte_of(p.y, k); }
                }
                *reinterpret_cast<uint2 *>(dst + y * stride) = make_uint2(pack4_sat_u8(v[0], v[1], v[2], v[3]), pack4_sat_u8(v[4], v[5], v[6], v[7]));
            }
            if (CLEAR) {
                uint4 *b = reinterpret_cast<uint4 *>(blocks) + i * 8;
#pragma unroll
                for (int y = 0; y < 8; y++) b[y] = make_uint4(0, 0, 0, 0);
            }
        }
        __syncwarp();                                        // this buffer is free for the load issued next iteration
    }
}

// put / put_signed / add pixels clamped (idctdsp.c:85-145): 16-byte row in, 8-byte row out.
// One thread per block row; a warp covers 4 blocks.  Purely HBM bound.
template <int MODE>
__global__ void __launch_bounds__(256)
pixels_clamped_kernel(const int16_t *__restrict__ blocks, uint8_t *__restrict__ frame,
                      const uint32_t *__restrict__ dst_off, ptrdiff_t stride, size_t n, int tiles_per_row)
{
    size_t t = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    size_t total = n * 8;
    for (; t < total; t += (size_t)gridDim.x * blockDim.x) {
        size_t i = t >> 3; int y = (int)(t & 7);
        uint4 r = ldg_stream(reinterpret_cast<const uint4 *>(blocks) + t);
        uint8_t *dst = frame + block_dst(dst_off, i, tiles_per_row, stride) + y * stride;
        int x[8] = { lo16s(r.x), hi16s(r.x), lo16s(r.y), hi16s(r.y), lo16s(r.z), hi16s(r.z), lo16s(r.w), hi16s(r.w) };
        if (MODE == 1) {
#pragma unroll
            for (int k = 0; k < 8; k++) x[k] += 128;
        } else if (MODE == 2) {
            uint2 p = *reinterpret_cast<const uint2 *>(dst);
#pragma unroll
            for (int k = 0; k < 4; k++) { x[k] += byte_of(p.x, k); x[4 + k] += byte_of(p.y, k); }
        }
        *reinterpret_cast<uint2 *>(dst) = make_uint2(pack4_sat_u8(x[0], x[1], x[2], x[3]), pack4_sat_u8(x[4], x[5], x[6], x[7]));
    }
}

__global__ void __launch_bounds__(256) clear_blocks_kernel(uint4 *__restrict__ p, size_t n16)
{
    size_t t = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    for (; t < n16; t += (size_t)gridDim.x * blockDim.x) p[t] = make_uint4(0, 0, 0, 0);
}

// fill_block_tab (blockdsp.c:39-58): rows of 16 or 8 identical bytes; records = (offset, value, h)
__global__ void __launch_bounds__(256)
fill_blocks_kernel(uint8_t *__restrict__ frame, const uint32_t *__restrict__ dst_off,
                   const uint8_t *__restrict__ value, ptrdiff_t stride, int h, int w16, size_t n)
{
    size_t t = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    size_t total = n * (size_t)h;
    for (; t < total; t += (size_t)gridDim.x * blockDim.x) {
        size_t i = t / (unsigned)h; int y = (int)(t - i * (unsigned)h);
        uint32_t v = value[i] * 0x01010101u;
        uint8_t *d = frame + dst_off[i] + y * stride;
        if (w16) *reinterpret_cast<uint4 *>(d) = make_uint4(v, v, v, v);
        else     *reinterpret_cast<uint2 *>(d) = make_uint2(v, v);
    }
}

static int grid_for(size_t work_items, int per_cta, int ctas_per_sm)
{
    size_t need = (work_items + per_cta - 1) / per_cta;
    size_t cap = (size_t)sm_count() * ctas_per_sm;
    if (need < 1) need = 1;
    return (int)(need < cap ? need : cap);
}

// cuTensorMapEncodeTiled through the runtime's driver entry point (the library does not link libcuda)
static bool make_block_tensor_map(CUtensorMap *tm, const int16_t *blocks, size_t n)
{
    typedef CUresult (*EncodeFn)(CUtensorMap *, CUtensorMapDataType, cuuint32_t, void *, const cuuint64_t *, const cuuint64_t *,
                                 const cuuint32_t *, const cuuint32_t *, CUtensorMapInterleave, CUtensorMapSwizzle,
                                 CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
    static EncodeFn fn = nullptr;
    static bool tried = false;
    if (!tried) {
        tried = true;
        void *p = nullptr;
        cudaDriverEntryPointQueryResult q;
        if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) == cudaSuccess && q == cudaDriverEntryPointSuccess) fn = (EncodeFn)p;
        else cudaGetLastError();
    }
    if (!fn) return false;
    const cuuint64_t dims[2] = { 64, (cuuint64_t)n }, strides[1] = { 128 };
    const cuuint32_t box[2] = { 64, 32 }, estr[2] = { 1, 1 };
    return fn(tm, CU_TENSOR_MAP_DATA_TYPE_UINT16, 2, (void *)blocks, dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
              CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) == CUDA_SUCCESS;
}

// the staged 8-bit IDCT with transform XF over n blocks; `who` names the entry point in error messages
template <class XF>
static int launch_idct8(const char *who, int mode, int16_t *blocks, uint8_t *frame, const uint32_t *dst_off, ptrdiff_t stride,
                        size_t n, int tiles_per_row, int clear, cudaStream_t st)
{
    if (n == 0) return 0;
    if (mode < 0 || mode > 2) { set_error_msg(who, "bad mode"); return -1; }
    if (mode != 2 && !dst_off && tiles_per_row <= 0) { set_error_msg(who, "need dst_off or tiles_per_row"); return -1; }
    size_t groups = (n + 31) / 32;
    // 16 CTAs per SM in the grid (about 3 waves of the 5 resident ones) rather than exactly one persistent wave: the shorter per-CTA
    // loops even out the tail
    int grid = grid_for(groups, IDCT_WARPS, 16);
    dim3 b(IDCT_WARPS * 32);
    // idct_put (the headline path) fetches through TMA; the cp.async fetch (same arithmetic, same throughput) serves unaligned block
    // arrays and drivers without a tensor-map encoder (idct_tma = 2 forces it: the parity tests run both fetches)
    if (mode == 0 && !clear && tuning("idct_tma") != 2 && !((uintptr_t)blocks & 15)) {
        CUtensorMap tm;
        if (make_block_tensor_map(&tm, blocks, n)) {
            simple_idct_kernel<0, false, 5, false, 0, true, XF><<<grid, b, 0, st>>>(blocks, frame, dst_off, stride, n, tiles_per_row, NoDq{}, tm);
            return check_launch(who);
        }
    }
    if (mode == 0) {
        if (clear) simple_idct_kernel<0, true, 5, false, 0, false, XF><<<grid, b, 0, st>>>(blocks, frame, dst_off, stride, n, tiles_per_row);
        else       simple_idct_kernel<0, false, 5, false, 0, false, XF><<<grid, b, 0, st>>>(blocks, frame, dst_off, stride, n, tiles_per_row);
    } else if (mode == 1) {
        if (clear) simple_idct_kernel<1, true, 5, false, 0, false, XF><<<grid, b, 0, st>>>(blocks, frame, dst_off, stride, n, tiles_per_row);
        else       simple_idct_kernel<1, false, 5, false, 0, false, XF><<<grid, b, 0, st>>>(blocks, frame, dst_off, stride, n, tiles_per_row);
    } else {
        simple_idct_kernel<2, false, 5, false, 0, false, XF><<<grid, b, 0, st>>>(blocks, frame, dst_off, stride, n, tiles_per_row);
    }
    return check_launch(who);
}

int launch_simple_idct(int mode, int16_t *blocks, uint8_t *frame, const uint32_t *dst_off, ptrdiff_t stride,
                       size_t n, int tiles_per_row, int clear, cudaStream_t st)
{
    return launch_idct8<SimpleIdct>("simple_idct_batch", mode, blocks, frame, dst_off, stride, n, tiles_per_row, clear, st);
}

// the Xvid IDCT through the same kernel: 16-byte aligned blocks and, for put / add, 8-byte aligned destinations (xvid_idct.cu decides)
int launch_xvid_idct_staged(int mode, int16_t *blocks, uint8_t *frame, const uint32_t *dst_off, ptrdiff_t stride,
                            size_t n, int tiles_per_row, int clear, cudaStream_t st)
{
    return launch_idct8<XvidIdct>("xvid_idct_batch", mode, blocks, frame, dst_off, stride, n, tiles_per_row, clear, st);
}

template <int KIND>
__global__ void __launch_bounds__(128)
mpeg_dequant_kernel(int16_t *__restrict__ blocks, const uint32_t *__restrict__ recs, size_t n, const DqTables T)
{
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const uint32_t rec = recs[i];
    if ((KIND == 1 || KIND == 4 || KIND == 6) && (int8_t)(rec >> 8) < 0) return;    // add_dequant_dct leaves such blocks alone
    const DqLane L = dq_lane<KIND>(rec, T);
    uint4 *b = reinterpret_cast<uint4 *>(blocks) + i * 8;
    int sum = -1;
#pragma unroll
    for (int r = 0; r < 8; r++) b[r] = dq_row<KIND>(b[r], r, T, L, sum);
}

int launch_mpeg_dequant(int kind, const DqTables &t, const uint32_t *recs, int16_t *blocks, size_t n, cudaStream_t st)
{
    if (n == 0) return 0;
    const int grid = (int)((n + 127) / 128);
    switch (kind) {
    case 0: mpeg_dequant_kernel<0><<<grid, 128, 0, st>>>(blocks, recs, n, t); break;
    case 1: mpeg_dequant_kernel<1><<<grid, 128, 0, st>>>(blocks, recs, n, t); break;
    case 2: mpeg_dequant_kernel<2><<<grid, 128, 0, st>>>(blocks, recs, n, t); break;
    case 3: mpeg_dequant_kernel<3><<<grid, 128, 0, st>>>(blocks, recs, n, t); break;
    case 4: mpeg_dequant_kernel<4><<<grid, 128, 0, st>>>(blocks, recs, n, t); break;
    case 5: mpeg_dequant_kernel<5><<<grid, 128, 0, st>>>(blocks, recs, n, t); break;
    case 6: mpeg_dequant_kernel<6><<<grid, 128, 0, st>>>(blocks, recs, n, t); break;
    default: set_error_msg("mpeg_dequant_batch", "bad kind"); return -1;
    }
    return check_launch("mpeg_dequant_batch");
}

// intra kinds run as idct_put, inter kinds as idct_add (put_dct / add_dequant_dct, libavcodec/mpegvideo.c:1401-1427)
template <class XF>
static int launch_dequant_idct8(const char *who, int kind, const DqTables &t, const uint32_t *recs, int16_t *blocks, uint8_t *frame,
                                const uint32_t *dst_off, ptrdiff_t stride, size_t n, int tiles_per_row, int clear, cudaStream_t st)
{
    if (n == 0) return 0;
    if (!dst_off && tiles_per_row <= 0) { set_error_msg(who, "need dst_off or tiles_per_row"); return -1; }
    const size_t groups = (n + 31) / 32;
    const int grid = grid_for(groups, IDCT_WARPS, 16);
    const dim3 b(IDCT_WARPS * 32);
    DqArgs a; a.recs = recs; a.t = t;
#define AVB_DQ(K, MODE) \
    case K: if (clear) simple_idct_kernel<MODE, true, 4, false, K + 1, false, XF><<<grid, b, 0, st>>>(blocks, frame, dst_off, stride, n, tiles_per_row, a); \
            else       simple_idct_kernel<MODE, false, 4, false, K + 1, false, XF><<<grid, b, 0, st>>>(blocks, frame, dst_off, stride, n, tiles_per_row, a); break;
    switch (kind) {
    AVB_DQ(0, 0) AVB_DQ(1, 1) AVB_DQ(2, 0) AVB_DQ(3, 0) AVB_DQ(4, 1) AVB_DQ(5, 0) AVB_DQ(6, 1)
    default: set_error_msg(who, "bad kind"); return -1;
    }
#undef AVB_DQ
    return check_launch(who);
}

int launch_mpeg_dequant_idct(int kind, const DqTables &t, const uint32_t *recs, int16_t *blocks, uint8_t *frame,
                             const uint32_t *dst_off, ptrdiff_t stride, size_t n, int tiles_per_row, int clear, cudaStream_t st)
{
    return launch_dequant_idct8<SimpleIdct>("mpeg_dequant_idct_batch", kind, t, recs, blocks, frame, dst_off, stride, n, tiles_per_row, clear, st);
}

int launch_mpeg_dequant_xvid_idct(int kind, const DqTables &t, const uint32_t *recs, int16_t *blocks, uint8_t *frame,
                                  const uint32_t *dst_off, ptrdiff_t stride, size_t n, int tiles_per_row, int clear, cudaStream_t st)
{
    return launch_dequant_idct8<XvidIdct>("mpeg_dequant_xvid_idct_batch", kind, t, recs, blocks, frame, dst_off, stride, n, tiles_per_row, clear, st);
}

// the staged FAAN IDCT: 16-byte aligned blocks and, for put / add, 8-byte aligned destinations (faan_idct.cu decides)
int launch_faan_idct_staged(int mode, int16_t *blocks, uint8_t *frame, const uint32_t *dst_off, ptrdiff_t stride,
                            size_t n, int tiles_per_row, int clear, cudaStream_t st)
{
    if (n == 0) return 0;
    const int grid = grid_for((n + 31) / 32, IDCT_WARPS, 16);
    const dim3 b(IDCT_WARPS * 32);
    if (mode == 0) {
        if (clear) faan_idct_kernel<0, true><<<grid, b, 0, st>>>(blocks, frame, dst_off, stride, n, tiles_per_row);
        else       faan_idct_kernel<0, false><<<grid, b, 0, st>>>(blocks, frame, dst_off, stride, n, tiles_per_row);
    } else if (mode == 1) {
        if (clear) faan_idct_kernel<1, true><<<grid, b, 0, st>>>(blocks, frame, dst_off, stride, n, tiles_per_row);
        else       faan_idct_kernel<1, false><<<grid, b, 0, st>>>(blocks, frame, dst_off, stride, n, tiles_per_row);
    } else {
        faan_idct_kernel<2, false><<<grid, b, 0, st>>>(blocks, frame, dst_off, stride, n, tiles_per_row);
    }
    return check_launch("faanidct_batch");
}

int launch_mpeg_dequant_faan_idct(int kind, const DqTables &t, const uint32_t *recs, int16_t *blocks, uint8_t *frame,
                                  const uint32_t *dst_off, ptrdiff_t stride, size_t n, int tiles_per_row, int clear, cudaStream_t st)
{
    static const char *who = "mpeg_dequant_faanidct_batch";
    if (n == 0) return 0;
    if (!dst_off && tiles_per_row <= 0) { set_error_msg(who, "need dst_off or tiles_per_row"); return -1; }
    const int grid = grid_for((n + 31) / 32, IDCT_WARPS, 16);
    const dim3 b(IDCT_WARPS * 32);
    DqArgs a; a.recs = recs; a.t = t;
#define AVB_DQ(K, MODE) \
    case K: if (clear) faan_idct_kernel<MODE, true, K + 1><<<grid, b, 0, st>>>(blocks, frame, dst_off, stride, n, tiles_per_row, a); \
            else       faan_idct_kernel<MODE, false, K + 1><<<grid, b, 0, st>>>(blocks, frame, dst_off, stride, n, tiles_per_row, a); break;
    switch (kind) {
    AVB_DQ(0, 0) AVB_DQ(1, 1) AVB_DQ(2, 0) AVB_DQ(3, 0) AVB_DQ(4, 1) AVB_DQ(5, 0) AVB_DQ(6, 1)
    default: set_error_msg(who, "bad kind"); return -1;
    }
#undef AVB_DQ
    return check_launch(who);
}

int launch_pixels_clamped(int mode, const int16_t *blocks, uint8_t *frame, const uint32_t *dst_off,
                          ptrdiff_t stride, size_t n, int tiles_per_row, cudaStream_t st)
{
    if (n == 0) return 0;
    if (!dst_off && tiles_per_row <= 0) { set_error_msg("pixels_clamped_batch", "need dst_off or tiles_per_row"); return -1; }
    int grid = grid_for(n * 8, 256, 8);
    switch (mode) {
    case 0: pixels_clamped_kernel<0><<<grid, 256, 0, st>>>(blocks, frame, dst_off, stride, n, tiles_per_row); break;
    case 1: pixels_clamped_kernel<1><<<grid, 256, 0, st>>>(blocks, frame, dst_off, stride, n, tiles_per_row); break;
    case 2: pixels_clamped_kernel<2><<<grid, 256, 0, st>>>(blocks, frame, dst_off, stride, n, tiles_per_row); break;
    default: set_error_msg("pixels_clamped_batch", "bad mode"); return -1;
    }
    return check_launch("pixels_clamped_batch");
}

int launch_clear_blocks(int16_t *blocks, size_t n_blocks, cudaStream_t st)
{
    if (n_blocks == 0) return 0;
    size_t n16 = n_blocks * 8;
    clear_blocks_kernel<<<grid_for(n16, 256, 8), 256, 0, st>>>(reinterpret_cast<uint4 *>(blocks), n16);
    return check_launch("clear_blocks_batch");
}

int launch_fill_blocks(uint8_t *frame, const uint32_t *dst_off, const uint8_t *value, ptrdiff_t stride, int h,
                       int w16, size_t n, cudaStream_t st)
{
    if (n == 0) return 0;
    fill_blocks_kernel<<<grid_for(n * h, 256, 8), 256, 0, st>>>(frame, dst_off, value, stride, h, w16, n);
    return check_launch("fill_blocks_batch");
}

}  // namespace avb
