// libav_b200/csrc/sws_fused_tma.cu -- same-size yuv420p -> rgb24 / bgr24 (the 4K benchmark geometry) with TMA-staged line buffers.
//
// Same arithmetic as sws_fused_rgb24_v3_kernel (swscale.cu): yuv2rgb24_X_c with a one-tap luma and a four-tap chroma bank
// (libswscale/output.c:936-995 + write :853-866), the line window of swscale() (swscale.c:450-616), the colour tables of yuv2rgb.c:633-658
// evaluated arithmetically.  What changes is how the bytes travel and how many instructions a pixel costs:
//   * a warp owns a 256 x 8 pixel tile (four row pairs).  Its luma rows (8 x 256 B) and the eight chroma lines of each plane that the
//     tile's vertical windows touch (8 x 128 B each) arrive by three cp.async.bulk.tensor (TMA, 3-D maps x / line / frame, zero fill
//     outside the plane) into one of the warp's own three stages and are awaited on that stage's mbarrier: no CTA-wide barrier exists
//     after start-up, the next two tiles are always in flight.  Warps are persistent: each takes its first FT_FIXED tiles by a fixed
//     stride over the tiles of all frames of the batch and the rest from a tile counter, so that all warps finish together.
//   * a thread owns 16 pixels x 4 rows (row pairs `half` and `half + 2` of the tile).  The seven chroma lines they need are
//     byte-transposed once (window 0-3), the windows of the next rows are one PRMT away (drop the oldest line, append the next); the
//     4-tap FIR is two IDP.2A on int16 taps.
//   * the rows leave through shared memory: four 768-byte rows per cp.async.bulk.tensor store (whole 128-byte lines per request).
//   * the per-(U, V) additive terms  cy * ((V * crv) >> 16) + kr,  cy * ((V * cgv) >> 16),  cy * ((U * cbu) >> 16) + kb,
//     cy * ((U * cgu) >> 16) + kg  come from two 256-entry tables in shared memory, built by the CTA from the context's constants
//     with exactly these formulas, 8 copies of each 8-byte entry so that every pair of lanes of a half-warp reads its own bank pair
//     (at most a 2-way bank conflict whatever the picture holds; 16 conflict-free copies leave no room for the third stage):
//     2 LDS.64 + 1 IADD instead of 12 integer instructions per chroma sample and row.
//   * luma loads and output stores carry an L2 evict-first policy: both are touched once, while the chroma lines are read again by the
//     next tile row.
//   * the launch is a programmatic dependent of the one before it on the stream: its CTAs build their tables while that launch drains,
//     and touch global memory only once it has completed.
//   * tiles at the top / bottom of the plane (clamped lines, shifted filters) and ragged last tiles take a row-by-row path with the
//     same per-row routine.
#include "sws_fused.h"
#include "tma.h"

namespace avb {

namespace {

constexpr int FT_STAGE = 4096;                  // Y 8 rows x 256 B | U 8 lines x 128 B | V 8 lines x 128 B
constexpr int FT_STAGES = 3;                    // tile stages per warp
// Tiles per warp by the fixed stride before the tile counter's.  The first ticket is drawn on the way to the last fixed tile: with
// only the pipeline's first tiles fixed, all warps draw it at once, in one burst on one address, at the start of the launch; 6, 8
// and 12 measured alike and about 1 % faster per step than 3 (profiles/README.md).
constexpr int FT_FIXED = 8;
static_assert(FT_FIXED >= 2, "the first ticket is drawn on the way to the last fixed tile");
constexpr int FT_OUT = 4 * 768;                 // output staging: four 768-byte rows (half a tile) per bulk tensor store
constexpr int FT_LUTC = 8;                      // lane copies of each term table entry
constexpr int FT_LUT_BYTES = 2 * 256 * FT_LUTC * 8;     // table by V {tr, tgv}, table by U {tb, tgu}: 256 entries x FT_LUTC copies x 8 B
constexpr int FT_MAX_WARPS = 12;                // the largest CTA
constexpr int FT_SMEM_MAX = 227 * 1024;         // shared memory a CTA may opt in to on sm_90
// The launch bound keeps the register budget of a 14-warp CTA, which the kernel's schedule was measured under (profiles/README.md):
// a 12-warp bound gives the same 127 registers but another instruction schedule.
constexpr int FT_BOUND_THREADS = 14 * 32;
constexpr int ft_smem_bytes(int warps) { return FT_LUT_BYTES + warps * (FT_STAGES * FT_STAGE + FT_OUT + 8 * FT_STAGES); }
static_assert(ft_smem_bytes(FT_MAX_WARPS) <= FT_SMEM_MAX, "the largest CTA's stages, slabs and tables must fit in shared memory");

struct FusedTmaArgs {
    uint8_t *dst; int dstStride; size_t dstFrame;
    int dstW, chrSrcH;
    int rp0, rowEnd;                  // first row pair of the launch (multiple of 4), first output row past it
    int tilesX, nTy;                  // tiles per tile row, tile rows of the launch
    int nitems;                       // nframes * nTy * tilesX
    int stepX, stepTy, stepF;         // the (tx, ty, frame) decomposition of the warp stride gridDim.x * warps
};

__device__ __forceinline__ int dp2a_lo(uint32_t k, uint32_t b, int c)
{ int d; asm("dp2a.lo.s32.u32 %0, %1, %2, %3;" : "=r"(d) : "r"(k), "r"(b), "r"(c)); return d; }
__device__ __forceinline__ int dp2a_hi(uint32_t k, uint32_t b, int c)
{ int d; asm("dp2a.hi.s32.u32 %0, %1, %2, %3;" : "=r"(d) : "r"(k), "r"(b), "r"(c)); return d; }

// lines r0..r3 hold 4 chroma columns each (one byte per column): out[c] = (r0.c, r1.c, r2.c, r3.c)
__device__ __forceinline__ void transpose4(uint32_t r0, uint32_t r1, uint32_t r2, uint32_t r3, uint32_t *out)
{
    const uint32_t t0 = __byte_perm(r0, r1, 0x5140), t1 = __byte_perm(r2, r3, 0x5140), t2 = __byte_perm(r0, r1, 0x7362), t3 = __byte_perm(r2, r3, 0x7362);
    out[0] = __byte_perm(t0, t1, 0x5410); out[1] = __byte_perm(t0, t1, 0x7632); out[2] = __byte_perm(t2, t3, 0x5410); out[3] = __byte_perm(t2, t3, 0x7632);
}
// the window one line lower: drop the oldest line, append column c of `next`
template <int C> __device__ __forceinline__ uint32_t slide(uint32_t w, uint32_t next) { return __byte_perm(w, next, ((4 + C) << 12) | 0x321); }
__device__ __forceinline__ void slide4(const uint32_t *w, uint32_t next, uint32_t *out)
{ out[0] = slide<0>(w[0], next); out[1] = slide<1>(w[1], next); out[2] = slide<2>(w[2], next); out[3] = slide<3>(w[3], next); }

// one output row of 16 pixels: TU / TV = the row's four chroma lines of each of the 8 chroma columns, yy = 16 luma bytes
template <bool BGR>
__device__ __forceinline__ void row16(const uint32_t (&TU)[8], const uint32_t (&TV)[8], uint32_t k01, uint32_t k23, uint4 yy,
                                      int cy, unsigned lutU_s, unsigned lutV_s, uint32_t (&o)[12])
{
#pragma unroll
    for (int q = 0; q < 4; q++) {                            // 4 pixels = 2 chroma columns per step
        const uint32_t yw = q == 0 ? yy.x : q == 1 ? yy.y : q == 2 ? yy.z : yy.w;
        int r[4], g[4], b[4];
#pragma unroll
        for (int e = 0; e < 2; e++) {
            const int c = 2 * q + e;
            // (2^18 + sum (u << 7) * coef) >> 19  ==  (2^11 + sum u * coef) >> 12
            const int su = dp2a_hi(k23, TU[c], dp2a_lo(k01, TU[c], 2048));
            const int sv = dp2a_hi(k23, TV[c], dp2a_lo(k01, TV[c], 2048));
            const int U = sat255(su >> 12), V = sat255(sv >> 12);        // per-value clip == the reference's flagged clip (host-checked range)
            const uint2 lv = lds64_ro(lutV_s + V * (FT_LUTC * 8)), lu = lds64_ro(lutU_s + U * (FT_LUTC * 8));
            const int tr = (int)lv.x, tb = (int)lu.x, tg = (int)(lu.y + lv.y);
            const int Ya = byte_of(yw, 2 * e), Yb = byte_of(yw, 2 * e + 1);
            r[2 * e] = cy * Ya + (BGR ? tb : tr); g[2 * e] = cy * Ya + tg; b[2 * e] = cy * Ya + (BGR ? tr : tb);
            r[2 * e + 1] = cy * Yb + (BGR ? tb : tr); g[2 * e + 1] = cy * Yb + tg; b[2 * e + 1] = cy * Yb + (BGR ? tr : tb);
        }
        o[3 * q + 0] = pack4_hi16_sat(r[0], g[0], b[0], r[1]);
        o[3 * q + 1] = pack4_hi16_sat(g[1], b[1], r[2], g[2]);
        o[3 * q + 2] = pack4_hi16_sat(b[2], r[3], g[3], b[3]);
    }
}

template <bool BGR>
__global__ void __launch_bounds__(FT_BOUND_THREADS, 1)
sws_fused_rgb24_tma_kernel(const RgbConstants k, const FusedTmaArgs a, const SwsPairTapsT *__restrict__ taps, int *tickets,
                           const __grid_constant__ CUtensorMap tmY, const __grid_constant__ CUtensorMap tmU, const __grid_constant__ CUtensorMap tmV,
                           const __grid_constant__ CUtensorMap tmD)
{
    extern __shared__ __align__(1024) uint8_t ft_smem[];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nwarps = blockDim.x >> 5;
    const unsigned smem_s = (unsigned)__cvta_generic_to_shared(ft_smem);
    const unsigned stage_s = smem_s + FT_LUT_BYTES + warp * FT_STAGES * FT_STAGE;
    const unsigned out_s = smem_s + FT_LUT_BYTES + nwarps * FT_STAGES * FT_STAGE + warp * FT_OUT;
    const unsigned mbar_s = smem_s + FT_LUT_BYTES + nwarps * (FT_STAGES * FT_STAGE + FT_OUT) + warp * 8 * FT_STAGES;

    // the two term tables, every entry FT_LUTC times (one copy per pair of lanes of a half-warp)
    uint2 *lut = reinterpret_cast<uint2 *>(ft_smem);
    for (int e = threadIdx.x; e < 2 * 256 * FT_LUTC; e += blockDim.x) {
        const int i = (e / FT_LUTC) & 255;
        uint2 val;
        if (e < 256 * FT_LUTC) { val.x = (uint32_t)(k.cy * ((i * k.crv) >> 16) + k.kr); val.y = (uint32_t)(k.cy * ((i * k.cgv) >> 16)); }
        else                   { val.x = (uint32_t)(k.cy * ((i * k.cbu) >> 16) + k.kb); val.y = (uint32_t)(k.cy * ((i * k.cgu) >> 16) + k.kg); }
        lut[e] = val;
    }
    if (lane == 0) {
#pragma unroll
        for (int s = 0; s < FT_STAGES; s++) mbar_init(mbar_s + 8 * s, 1);
        mbar_init_fence();
    }
    __syncthreads();
    // Launched as a programmatic dependent of the previous launch on the stream, the CTA gets here (tables built, barriers set up)
    // while that launch drains; nothing in global memory is touched before it has completed.
    asm volatile("griddepcontrol.wait;" ::: "memory");
    asm volatile("griddepcontrol.launch_dependents;" ::: "memory");

    const int cg = lane & 15, half = lane >> 4;
    const unsigned lutV_s = smem_s + (cg % FT_LUTC) * 8, lutU_s = smem_s + 256 * FT_LUTC * 8 + (cg % FT_LUTC) * 8;

    const int item = blockIdx.x * nwarps + warp;
    if (item >= a.nitems) return;
    const int wstride = gridDim.x * nwarps;
    const uint64_t evict_first = l2_policy_evict_first();
    auto advance = [&](int &tx, int &ty, int &f) {
        tx += a.stepX; f += a.stepF;
        if (tx >= a.tilesX) { tx -= a.tilesX; ty++; }
        ty += a.stepTy;
        if (ty >= a.nTy) { ty -= a.nTy; f++; }
    };
    auto tile_words = [&](int ty) { return __ldg(reinterpret_cast<const int2 *>(&taps[a.rp0 + 4 * ty].base)); };   // (base, interior)
    // A warp's first FT_FIXED tiles are fixed (item + s * wstride); the rest are handed out by the ticket counter in order (tx, then
    // tile row, then frame), so that a warp that runs faster takes more tiles and the warps end together.  Lane 0 draws each ticket
    // one tile before the warp reads it.  Every warp draws until it gets a ticket past the last tile, once; the warp that draws the
    // last of those wstride failing tickets puts the counter back to 0 for the next launch on the stream, which reads it only after
    // its own griddepcontrol.wait.
    const long long nfixed = (long long)FT_FIXED * wstride;
    const bool dyn = a.nitems > nfixed;
    const int nlast = dyn ? (int)(a.nitems - nfixed) + wstride - 1 : 0;
    auto issue = [&](int tx, int ty, int f, int base, unsigned st) {
        if (lane == 0) {
            const unsigned mb = mbar_s + 8 * st, dst = stage_s + st * FT_STAGE;
            fence_proxy_async();                              // the stage was last read by ordinary shared loads
            mbar_expect_tx(mb, FT_STAGE);
            tma_load_3d_hint(dst, &tmY, tx * 256, 2 * (a.rp0 + 4 * ty), f, mb, evict_first);
            tma_load_3d(dst + 2048, &tmU, tx * 128, base, f, mb);
            tma_load_3d(dst + 3072, &tmV, tx * 128, base, f, mb);
        }
    };
    // The tile issued next (n, FT_STAGES - 1 tiles ahead) is tracked by item and coordinates; the table words of n are fetched a whole
    // tile before its loads are issued; the items and words of the tiles in flight are kept in qi and q (oldest first).
    int ntx = item % a.tilesX, nty, nf;
    { const int t2 = item / a.tilesX; nty = t2 % a.nTy; nf = t2 / a.nTy; }
    long long nitem = item;
    int ticket = 0;                                   // lane 0: the ticket drawn ahead
    auto next = [&]() {
        if (!dyn || nitem < nfixed - 2 * wstride) { nitem += wstride; advance(ntx, nty, nf); }
        else if (nitem < nfixed - wstride) {          // on to the last fixed tile: draw the first ticket
            nitem += wstride; advance(ntx, nty, nf);
            if (lane == 0) ticket = atomicAdd(tickets, 1);
        } else if (nitem < a.nitems) {
            const int t = __shfl_sync(0xffffffffu, ticket, 0);
            nitem = nfixed + t;
            if (nitem < a.nitems) {
                ntx = (int)(nitem % a.tilesX);
                const int t2 = (int)(nitem / a.tilesX); nty = t2 % a.nTy; nf = t2 / a.nTy;
                if (lane == 0) ticket = atomicAdd(tickets, 1);
            } else if (t == nlast && lane == 0) {
                atomicExch(tickets, 0);
            }
        }
    };
    int2 q[FT_STAGES - 1];
    int qi[FT_STAGES - 1];
#pragma unroll
    for (int s = 0; s < FT_STAGES - 1; s++) {
        qi[s] = (int)min(nitem, (long long)a.nitems);
        q[s] = nitem < a.nitems ? tile_words(nty) : make_int2(0, 0);
        if (nitem < a.nitems) issue(ntx, nty, nf, q[s].x, s);
        next();
    }
    int2 nw = nitem < a.nitems ? tile_words(nty) : make_int2(0, 0);

    unsigned st = 0, phase = 0;
    while (qi[0] < a.nitems) {
        const int2 cw = q[0];
        const int ctx = qi[0] % a.tilesX, ct2 = qi[0] / a.tilesX, cty = ct2 % a.nTy, cf = ct2 / a.nTy;
        // the stage computed last (st - 1) is free again: the tile FT_STAGES - 1 tiles ahead starts travelling before this one is touched
        if (nitem < a.nitems) issue(ntx, nty, nf, nw.x, st == 0 ? FT_STAGES - 1 : st - 1);
#pragma unroll
        for (int s = 0; s < FT_STAGES - 2; s++) { q[s] = q[s + 1]; qi[s] = qi[s + 1]; }
        q[FT_STAGES - 2] = nw; qi[FT_STAGES - 2] = (int)min(nitem, (long long)a.nitems);
        next();
        nw = nitem < a.nitems ? tile_words(nty) : make_int2(0, 0);

        const int rpT = a.rp0 + 4 * cty;
        mbar_wait(mbar_s + 8 * st, phase);                                       // the k-th use of a stage completes its phase k
        const unsigned sY = stage_s + st * FT_STAGE, sU = sY + 2048, sV = sY + 3072;
        // Rows leave the warp four at a time: the half-warps' first pairs are tile rows 0-3, their second pairs rows 4-7.  A row is staged
        // in a 4 x 768-byte slab of the warp; one bulk tensor store writes the four rows (whole 128-byte lines: three 16-byte STG per lane
        // 48 bytes apart cost twice the L1 -> L2 write transactions, measured).  Columns past the width / rows past the range are clipped
        // by the tensor map.
        auto stage_row = [&](int slot, const uint32_t (&o)[12]) {
#pragma unroll
            for (int j = 0; j < 3; j++) sts128(out_s + slot * 768 + cg * 48 + 16 * j, make_uint4(o[4 * j], o[4 * j + 1], o[4 * j + 2], o[4 * j + 3]));
        };
        auto slab_free = [&]() { if (lane == 0) bulk_wait_read<0>(); __syncwarp(); };       // the previous store has read the slab
        auto flush = [&](int g) {
            fence_proxy_async();
            __syncwarp();
            if (lane == 0) {
                tma_store_3d_hint(&tmD, ctx * 192, 2 * rpT + 4 * g, cf, out_s, evict_first);
                bulk_commit();
            }
        };

        if (cw.y) {
            // interior tile: pair q of the tile filters chroma lines q .. q + 3 (first row) and q + 1 .. q + 4 (second row) of the stage.
            // This thread's pairs are `half` and `half + 2`: seven lines, four windows one line apart
            uint4 yy[4];
            uint2 ul[7], vl[7];
#pragma unroll
            for (int r = 0; r < 4; r++) yy[r] = lds128(sY + (2 * half + (r & 1) + 4 * (r >> 1)) * 256 + cg * 16);
#pragma unroll
            for (int j = 0; j < 7; j++) { ul[j] = lds64(sU + (half + j) * 128 + cg * 8); vl[j] = lds64(sV + (half + j) * 128 + cg * 8); }
            const uint4 tA = __ldg(reinterpret_cast<const uint4 *>(taps + rpT + half)), tB = __ldg(reinterpret_cast<const uint4 *>(taps + rpT + half + 2));
            __syncwarp();
            uint32_t WU[8], WV[8], XU[8], XV[8], o[12];
            transpose4(ul[0].x, ul[1].x, ul[2].x, ul[3].x, WU); transpose4(ul[0].y, ul[1].y, ul[2].y, ul[3].y, WU + 4);
            transpose4(vl[0].x, vl[1].x, vl[2].x, vl[3].x, WV); transpose4(vl[0].y, vl[1].y, vl[2].y, vl[3].y, WV + 4);
            slab_free();
            row16<BGR>(WU, WV, tA.x, tA.y, yy[0], k.cy, lutU_s, lutV_s, o); stage_row(2 * half, o);
            slide4(WU, ul[4].x, XU); slide4(WU + 4, ul[4].y, XU + 4); slide4(WV, vl[4].x, XV); slide4(WV + 4, vl[4].y, XV + 4);
            row16<BGR>(XU, XV, tA.z, tA.w, yy[1], k.cy, lutU_s, lutV_s, o); stage_row(2 * half + 1, o);
            flush(0);
            slide4(XU, ul[5].x, WU); slide4(XU + 4, ul[5].y, WU + 4); slide4(XV, vl[5].x, WV); slide4(XV + 4, vl[5].y, WV + 4);
            row16<BGR>(WU, WV, tB.x, tB.y, yy[2], k.cy, lutU_s, lutV_s, o);
            slab_free();
            stage_row(2 * half, o);
            slide4(WU, ul[6].x, XU); slide4(WU + 4, ul[6].y, XU + 4); slide4(WV, vl[6].x, XV); slide4(WV + 4, vl[6].y, XV + 4);
            row16<BGR>(XU, XV, tB.z, tB.w, yy[3], k.cy, lutU_s, lutV_s, o); stage_row(2 * half + 1, o);
            flush(1);
        } else {
            // plane edges and ragged tiles: every row fetches its own four (clamped) lines
#pragma unroll 1
            for (int r = 0; r < 4; r++) {
                const int trow = 2 * half + (r & 1) + 4 * (r >> 1);
                const int row = min(2 * rpT + trow, a.rowEnd - 1);               // rows past the launch's range compute a discarded duplicate: the loop stays warp-uniform
                const SwsPairTapsT *t = taps + (row >> 1);
                const uint2 kk = __ldg(reinterpret_cast<const uint2 *>(t) + (row & 1));
                const int first = __ldg(&t->first0 + (row & 1));
                uint2 ul[4], vl[4];
#pragma unroll
                for (int j = 0; j < 4; j++) {
                    const int line = min(max(min(max(first + j, 0), a.chrSrcH - 1) - cw.x, 0), 7);   // 0..7 (host-checked for rows inside the range)
                    ul[j] = lds64(sU + line * 128 + cg * 8); vl[j] = lds64(sV + line * 128 + cg * 8);
                }
                const uint4 yy = lds128(sY + trow * 256 + cg * 16);
                uint32_t TU[8], TV[8], o[12];
                transpose4(ul[0].x, ul[1].x, ul[2].x, ul[3].x, TU); transpose4(ul[0].y, ul[1].y, ul[2].y, ul[3].y, TU + 4);
                transpose4(vl[0].x, vl[1].x, vl[2].x, vl[3].x, TV); transpose4(vl[0].y, vl[1].y, vl[2].y, vl[3].y, TV + 4);
                row16<BGR>(TU, TV, kk.x, kk.y, yy, k.cy, lutU_s, lutV_s, o);
                if (!(r & 1)) slab_free();
                stage_row(trow & 3, o);
                if (r & 1) flush(r >> 1);
            }
            __syncwarp();
        }
        if (++st == FT_STAGES) { st = 0; phase ^= 1u; }
    }
    if (lane == 0) bulk_wait<0>();
}

}  // namespace

int sws_fused_tma_launch(const RgbConstants &k, int bgr, int dstW, int dstH, int chrSrcW, int chrSrcH, const FusedArgs &a,
                         const SwsPairTapsT *taps, int *tickets, int nframes, cudaStream_t st)
{
    const int pairs = dstH / 2;
    const int rp0 = a.rp0, rp1 = a.rp1 < pairs ? a.rp1 : pairs;
    if (nframes <= 0 || rp1 <= rp0) return 0;
    // what a tensor map can describe: 16-byte aligned planes and pitches; tiles are aligned to multiples of four row pairs
    if ((rp0 & 3) || ((rp1 & 3) && rp1 != pairs)) return 1;
    if (((uintptr_t)a.y | (uintptr_t)a.u | (uintptr_t)a.v | (uintptr_t)a.dst) & 15) return 1;
    if ((a.yStride | a.uStride | a.vStride | a.dstStride) & 15) return 1;
    if (nframes > 1 && ((a.yFrame | a.uFrame | a.vFrame | a.dstFrame) & 15)) return 1;
    if (a.yStride <= 0 || a.uStride <= 0 || a.vStride <= 0) return 1;
    CUtensorMap tmY, tmU, tmV, tmD;
    {
        // the destination as 32-bit words: a 256-pixel row of a tile is 768 bytes = 192 words (a box side is at most 256 elements)
        const cuuint64_t dD[3] = { (cuuint64_t)dstW * 3 / 4, (cuuint64_t)(2 * rp1), (cuuint64_t)nframes };
        const cuuint64_t sD[2] = { (cuuint64_t)a.dstStride, nframes > 1 ? (cuuint64_t)a.dstFrame : (cuuint64_t)a.dstStride * dstH };
        const cuuint32_t bD[3] = { 192, 4, 1 };
        if (a.dstStride <= 0 || !tma_encode(&tmD, CU_TENSOR_MAP_DATA_TYPE_UINT32, 3, a.dst, dD, sD, bD)) return 1;
        const cuuint64_t dY[3] = { (cuuint64_t)dstW, (cuuint64_t)dstH, (cuuint64_t)nframes };
        const cuuint64_t dC[3] = { (cuuint64_t)chrSrcW, (cuuint64_t)chrSrcH, (cuuint64_t)nframes };
        const cuuint64_t sY[2] = { (cuuint64_t)a.yStride, nframes > 1 ? (cuuint64_t)a.yFrame : (cuuint64_t)a.yStride * dstH };
        const cuuint64_t sU[2] = { (cuuint64_t)a.uStride, nframes > 1 ? (cuuint64_t)a.uFrame : (cuuint64_t)a.uStride * chrSrcH };
        const cuuint64_t sV[2] = { (cuuint64_t)a.vStride, nframes > 1 ? (cuuint64_t)a.vFrame : (cuuint64_t)a.vStride * chrSrcH };
        const cuuint32_t bY[3] = { 256, 8, 1 }, bC[3] = { 128, 8, 1 };
        if (!tma_encode(&tmY, CU_TENSOR_MAP_DATA_TYPE_UINT8, 3, a.y, dY, sY, bY) ||
            !tma_encode(&tmU, CU_TENSOR_MAP_DATA_TYPE_UINT8, 3, a.u, dC, sU, bC) ||
            !tma_encode(&tmV, CU_TENSOR_MAP_DATA_TYPE_UINT8, 3, a.v, dC, sV, bC)) return 1;
    }
    FusedTmaArgs fa;
    fa.dst = a.dst; fa.dstStride = a.dstStride; fa.dstFrame = a.dstFrame;
    fa.dstW = dstW; fa.chrSrcH = chrSrcH;
    fa.rp0 = rp0; fa.rowEnd = 2 * rp1;
    fa.tilesX = (dstW + 255) / 256; fa.nTy = (rp1 - rp0 + 3) / 4;
    const long long nitems = (long long)nframes * fa.nTy * fa.tilesX;
    if (nitems > 0x7fffffff / 2) return 1;
    fa.nitems = (int)nitems;

    // 12 warps per CTA (one CTA per SM); batches of fewer than two tiles per warp of that grid take 4-warp CTAs, which spread them over
    // more SMs
    const int warps = nitems >= 12 * 2 * sm_count() ? 12 : 4;
    const int smem = ft_smem_bytes(warps);
    const int b = bgr ? 1 : 0;
    auto kern = b ? sws_fused_rgb24_tma_kernel<true> : sws_fused_rgb24_tma_kernel<false>;
    static int attr_smem[2] = {};                   // the largest dynamic shared memory each kernel has been allowed so far
    static int ctas_per_sm[2][FT_MAX_WARPS + 1] = {};
    if (smem > attr_smem[b]) {
        if (cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, smem) != cudaSuccess) {
            set_error("sws_scale:fused tma", cudaGetLastError()); return -1;
        }
        attr_smem[b] = smem;
    }
    if (!ctas_per_sm[b][warps]) {
        int n = 0;
        if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&n, kern, warps * 32, smem) != cudaSuccess || n <= 0) {
            set_error_msg("sws_scale:fused tma", "kernel shape does not fit an SM"); cudaGetLastError(); return -1;
        }
        ctas_per_sm[b][warps] = n;
    }
    // the grid (no more CTAs than the work can use) and the (tx, ty, frame) steps of the warp stride
    const long long max_ctas = (nitems + warps - 1) / warps;
    long long grid = (long long)sm_count() * ctas_per_sm[b][warps];
    if (grid > max_ctas) grid = max_ctas;
    const long long wstride = grid * warps;
    fa.stepX = (int)(wstride % fa.tilesX);
    { const long long t2 = wstride / fa.tilesX; fa.stepTy = (int)(t2 % fa.nTy); fa.stepF = (int)(t2 / fa.nTy); }
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = dim3((unsigned)grid); cfg.blockDim = dim3(warps * 32); cfg.dynamicSmemBytes = smem; cfg.stream = st;
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[0].val.programmaticStreamSerializationAllowed = 1;
    cfg.attrs = attr; cfg.numAttrs = 1;
    if (cudaLaunchKernelEx(&cfg, kern, k, fa, taps, tickets, tmY, tmU, tmV, tmD) != cudaSuccess) { set_error("sws_scale:fused tma", cudaGetLastError()); return -1; }
    return check_launch("sws_scale:fused tma");
}

}  // namespace avb
