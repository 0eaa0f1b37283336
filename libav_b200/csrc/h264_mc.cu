// libav_b200/csrc/h264_mc.cu -- batched H.264 inter prediction (config 3's first stage): work distribution around mc_block().
//
// The unit of work is a 4x4 luma block (+ its 2x2 chroma blocks): every partition size of the standard is a whole number of them, and
// one thread finishes one (h264_mc_block.cuh).  A warp takes 32 consecutive records, counts their blocks with a shuffle scan, and
// walks the 32 .. 512 blocks 32 at a time; a lane finds its (record, block) by a five-step search of the warp's offset table in
// shared memory.  Lanes of one partition share the quarter-sample position, so on real streams a warp needs few of the components
// F / H / V / J; which ones is voted per 32 blocks.  `put` records run in pass 0, `avg` records (second prediction direction,
// h264_mb.c:322-366) in pass 1 -- two ordered launches keep put-before-avg without ordering the records themselves.
#include "h264_mc_block.cuh"
#include <type_traits>
#include "../../include/avdsp_b200.h"

namespace avb {

namespace {

__global__ void __launch_bounds__(128, 6)
h264_mc_kernel_v2(const FFH264MCRecord *__restrict__ recs, size_t n, const FFH264RefPlanes *__restrict__ refs,
                  uint8_t *__restrict__ dy, uint8_t *__restrict__ dcb, uint8_t *__restrict__ dcr, int ls, int uvls, int pw, int ph, int pass)
{
    __shared__ int s_off[4][33];
    __shared__ uint16_t s_edge[4][64];                     // deferred edge blocks (ordinals)
    __shared__ const uint8_t *s_pl[4][32][3];               // the record's reference planes (read once per record, not once per block)
    __shared__ uint32_t s_rec[4][32][4];                   // x | y << 16, mvx | mvy << 16, w | h << 8 | avg << 16 | ref << 24, first luma row of the record's picture
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const size_t r0 = ((size_t)blockIdx.x * 4 + warp) * 32;
    if (r0 >= n) return;
    int nb = 0;
    {
        uint32_t w0 = 0, w1 = 0, w2 = 0, ly0 = 0;
        if (r0 + lane < n) {
            const uint32_t *p = reinterpret_cast<const uint32_t *>(recs + r0 + lane);
            w0 = __ldg(p); w1 = __ldg(p + 1); w2 = __ldg(p + 2);
            const int w = w2 & 255, h = (w2 >> 8) & 255, avg = (w2 >> 16) & 255;
            if ((avg != 0) == (pass != 0)) nb = (w >> 2) * (h >> 2);
            ly0 = (uint32_t)(((int)(int16_t)(w0 >> 16) / ph) * ph);
            if (nb) {
                const FFH264RefPlanes rp = refs[w2 >> 24];
                s_pl[warp][lane][0] = rp.y; s_pl[warp][lane][1] = rp.cb; s_pl[warp][lane][2] = rp.cr;
            }
        }
        s_rec[warp][lane][0] = w0; s_rec[warp][lane][1] = w1; s_rec[warp][lane][2] = w2; s_rec[warp][lane][3] = ly0;
    }
    int incl = nb;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) { const int v = __shfl_up_sync(0xffffffffu, incl, d); if (lane >= d) incl += v; }
    s_off[warp][lane] = incl - nb;
    const int total = __shfl_sync(0xffffffffu, incl, 31);
    if (lane == 0) s_off[warp][32] = total;
    __syncwarp();

    // one block: ordinal q of the warp's blocks -> (record, block) -> mc_block
    auto run = [&](int q, bool live, auto edge_tag) {
        constexpr bool EDGE = decltype(edge_tag)::value;
        // the last record whose first block is <= q (records without blocks in this pass share their successor's offset)
        int j = 0;
        if (live) {
#pragma unroll
            for (int step = 16; step; step >>= 1) if (s_off[warp][j + step] <= q) j += step;
        }
        const uint32_t w0 = s_rec[warp][j][0], w1 = s_rec[warp][j][1], w2 = s_rec[warp][j][2];
        const int ly0 = (int)s_rec[warp][j][3];
        const int rx = (int16_t)(w0 & 0xffff), ry = (int16_t)(w0 >> 16), mvx = (int16_t)(w1 & 0xffff), mvy = (int16_t)(w1 >> 16);
        const int rw = w2 & 255, avg = (w2 >> 16) & 255;
        const int b = q - s_off[warp][j], bw = rw >> 2;
        const int by = bw == 4 ? b >> 2 : bw == 2 ? b >> 1 : b, bx = b - by * bw;
        const int x = rx + 4 * bx, y = ry + 4 * by, mx = mvx + 4 * x, my = mvy + 4 * y;
        const int fx = mx & 3, fy = my & 3;
        McPlanes pl = { nullptr, nullptr, nullptr };
        bool inside = false;
        if (live) {
            pl.y = s_pl[warp][j][0]; pl.cb = s_pl[warp][j][1]; pl.cr = s_pl[warp][j][2];
            const bool aligned = !(((uintptr_t)pl.y | (uintptr_t)pl.cb | (uintptr_t)pl.cr | (uintptr_t)ls | (uintptr_t)uvls) & 3);
            inside = mc_block_inside(pw, ph, ly0, mx, my, aligned);
        }
        const bool mine = live && (EDGE || inside);                   // (the interior pass leaves edge blocks to the deferred pass)
        const bool uj = mine && ((fx == 2 && fy != 0) || (fy == 2 && fx != 0));
        const bool uh = mine && fx != 0 && fy != 2;                   // H: fy == 0, or both odd, or fx == 2 with fy odd
        const bool uv = mine && fy != 0 && fx != 2;                   // V: fx == 0, or both odd, or fy == 2 with fx odd
        const bool need_j = __any_sync(0xffffffffu, uj), need_h = __any_sync(0xffffffffu, uh), need_v = __any_sync(0xffffffffu, uv);
        if (mine) mc_block<EDGE>(pl, dy, dcb, dcr, ls, uvls, pw, ph, ly0, x, y, mx, my, avg, need_h, need_v, need_j);
        return live && !inside;
    };

    // Blocks whose patches leave the picture (or whose planes are unaligned) fetch sample by sample.  They are few, but a warp that
    // mixed them with interior blocks would execute both fetch paths for everyone: they are set aside and run 32 at a time.
    int ne = 0;
    auto run_deferred = [&](int count) {
        const int q = lane < count ? (int)s_edge[warp][lane] : 0;
        run(q, lane < count, std::true_type());
    };
    for (int q0 = 0; q0 < total; q0 += 32) {
        const int q = q0 + lane;
        const bool edge = run(q, q < total, std::false_type());
        const unsigned em = __ballot_sync(0xffffffffu, edge);
        if (edge) s_edge[warp][ne + __popc(em & ((1u << lane) - 1u))] = (uint16_t)q;
        ne += __popc(em);
        __syncwarp();
        if (ne >= 32) {
            run_deferred(32);
            __syncwarp();
            const uint16_t keep = lane < ne - 32 ? s_edge[warp][32 + lane] : (uint16_t)0;
            __syncwarp();
            if (lane < ne - 32) s_edge[warp][lane] = keep;
            ne -= 32;
            __syncwarp();
        }
    }
    if (ne > 0) run_deferred(ne);
}

}  // namespace

// 0 launched, 1 not applicable (destination planes the word stores cannot address): the caller runs the byte-wise kernel
int launch_h264_mc_v2(const FFH264MCRecord *recs, size_t n, const FFH264RefPlanes *refs, uint8_t *dy, uint8_t *dcb, uint8_t *dcr,
                      int ls, int uvls, int pw, int ph, cudaStream_t st)
{
    if (((uintptr_t)dy | (uintptr_t)ls) & 3) return 1;
    if (((uintptr_t)dcb | (uintptr_t)dcr | (uintptr_t)uvls) & 1) return 1;
    if (ph <= 0 || (ph & 1) || (pw & 1)) return 1;
    const unsigned grid = (unsigned)((n + 127) / 128);
    // compiled for 6 resident CTAs per SM (80 registers, ~40 words of spill that stay in L1): the kernel waits on its patch loads, so warps
    // in flight count for more than registers, up to the point where spills cost more -- bench.py --workload h264 on an H100 80GB HBM3
    // (700 W): 4 CTAs (128 registers) 3.85 ms per step, 6 CTAs 3.76 ms, 8 CTAs (64 registers, ~110 words of spill) 4.09 ms.
    for (int pass = 0; pass < 2; pass++) h264_mc_kernel_v2<<<grid, 128, 0, st>>>(recs, n, refs, dy, dcb, dcr, ls, uvls, pw, ph, pass);
    return check_launch("h264_mc_batch") ? -1 : 0;
}

}  // namespace avb
