// libav_b200/csrc/h264_hbd_batch.cu -- the batched H.264 calls for 9 / 10-bit pictures (uint16 samples, int32 coefficients: the
// BIT_DEPTH > 8 instances of libavcodec/bit_depth_template.c:49-67) and for chroma_format_idc 2 (4:2:2) content:
//
//   ff_h264_idct_add_mb_batch_hbd_cuda   h264_idct_add16 / add16intra / idct8_add4 / idct_add8 / idct_add8_422 per macroblock
//                                        (libavcodec/h264idct_template.c:174-236), 4:2:0 and 4:2:2
//   ff_h264_mc_batch_hbd_cuda            mc_dir_part() (libavcodec/h264_mb.c:204-320): H264QpelContext + H264ChromaContext put / avg with
//                                        emulated_edge_mc, 4:2:0 and 4:2:2 (chroma rows at full vertical resolution, :287-316)
//   ff_h264_deblock_batch_hbd_cuda       the loop filters of libavcodec/h264dsp_template.c:104-328 over whole pictures in the reference's
//                                        serial raster order (h264_loopfilter.c:397-415), 4:2:0
//
// These are the FUNCTIONAL batched paths for that content, built from the per-sample arithmetic of h264dsp_hbd.cuh (the one the table
// slots of slots_hbd.cu use); they are not shaped like the 8-bit kernels (h264_mc.cu / h264_residual.cu / h264_deblock.cu), which
// live on packed bytes.  Mapping:
//   residual   warp per macroblock, lane per transform block exactly as the C dispatchers iterate (lanes never communicate)
//   MC         warp per partition record, lanes stride over its luma and chroma samples, every reference sample through a clamped fetch
//              (= emulated_edge_mc); `put` records in pass 0, `avg` records in pass 1 (two ordered launches)
//   deblock    one CTA per picture and plane kind (luma; cb + cr), its warps take macroblock rows round-robin and run them as a wavefront (a
//              row stays two macroblocks behind the row above): progress counters live in SHARED memory, so no inter-CTA ordering, fence
//              or dispatch-order assumption exists; all warps of a CTA are resident, rows are taken in increasing order, hence no
//              deadlock.  Within a macroblock: 16 lanes filter the vertical edges line by line, then the horizontal ones column by column
//              (h264_loopfilter.c:238-395 order per plane); the next macroblock's record and sample rows are prefetched meanwhile.
// A picture of a batch starts `pic_h` luma rows after the previous one in the same planes (like the 8-bit calls).
#include "h264dsp.cuh"
#include "h264dsp_hbd.cuh"
#include "h264pred_hbd.cuh"
#include "../../include/avdsp_b200.h"

namespace avb {

namespace {

using hbd::px;

// the transforms by sample type: 9 / 10 bit = h264dsp_hbd.cuh (uint16 samples, int32 coefficients), 8 bit = h264dsp.cuh (uint8, int16; the 4:2:2
// pictures: 8-bit 4:2:0 has its own kernels in h264_residual.cu)
template <typename PX> struct Transform;
template <> struct Transform<uint16_t> {
    typedef int32_t coef;
    static __device__ __forceinline__ void idct4(int bits, uint16_t *d, coef *b, int st) { hbd::idct4_add(bits, d, b, st); }
    static __device__ __forceinline__ void idct8(int bits, uint16_t *d, coef *b, int st) { hbd::idct8_add(bits, d, b, st); }
    static __device__ __forceinline__ void dc(int bits, uint16_t *d, coef *b, int st, int n) { hbd::dc_add(bits, d, b, st, n); }
};
template <> struct Transform<uint8_t> {
    typedef int16_t coef;
    static __device__ __forceinline__ void idct4(int, uint8_t *d, coef *b, int st) { h264_idct4_add(d, b, st); }
    static __device__ __forceinline__ void idct8(int, uint8_t *d, coef *b, int st) { h264_idct8_add(d, b, st); }
    static __device__ __forceinline__ void dc(int, uint8_t *d, coef *b, int st, int n) { h264_dc_add(d, b, st, n); }
};

// ---------------------------------------------------------------------------------------------------------------------------------
template <typename PX>
__global__ void __launch_bounds__(128)
h264_residual_hbd_kernel(int bits, int c422, const FFH264ResidualMB *__restrict__ mbs, size_t n, typename Transform<PX>::coef *__restrict__ coeffs, size_t coeff_stride,
                         const uint8_t *__restrict__ nnzc, uint8_t *__restrict__ luma, uint8_t *__restrict__ cb, uint8_t *__restrict__ cr, int ls, int uvls)
{
    typedef Transform<PX> T;
    const int lane = threadIdx.x & 31;
    const size_t mb = (size_t)blockIdx.x * 4 + (threadIdx.x >> 5);
    if (mb >= n) return;
    const FFH264ResidualMB r = mbs[mb];
    typename T::coef *gc = coeffs + mb * coeff_stride;
    const uint8_t *nz = nnzc + mb * 120;
    const int lsp = ls / (int)sizeof(PX), uvlsp = uvls / (int)sizeof(PX);                     // row distance in samples
    if (lane < 16) {
        if (r.luma_mode > 2) return;
        const int i = lane;
        PX *d = reinterpret_cast<PX *>(luma + r.luma_off) + blk_x(i) + (size_t)blk_y(i) * lsp;
        typename T::coef *b = gc + 16 * i;
        const int nnz = nz[scan8_of(i)];
        if (r.luma_mode == 0)      { if (nnz) { if (nnz == 1 && b[0]) T::dc(bits, d, b, lsp, 4); else T::idct4(bits, d, b, lsp); } }       // :174-183
        else if (r.luma_mode == 1) { if (nnz) T::idct4(bits, d, b, lsp); else if (b[0]) T::dc(bits, d, b, lsp, 4); }                       // :185-191
        else if ((i & 3) == 0 && nnz) { if (nnz == 1 && b[0]) T::dc(bits, d, b, lsp, 8); else T::idct8(bits, d, b, lsp); }                 // :193-202
    } else if (r.chroma) {
        // 4:2:0 (:204-214): blocks 16..19 / 32..35.  4:2:2 (:216-236): eight per plane; the lower four keep their coefficients at block i
        // but are addressed through scan8[i + 4] / block_offset[i + 4] (rows 8..15 of the 8 x 16 chroma macroblock)
        const int per = c422 ? 8 : 4, t = lane - 16;
        if (t >= 2 * per) return;
        const int plane = t / per, k = t % per, i = 16 + 16 * plane + k, e = k >= 4 ? i + 4 : i, ke = e & 15;
        PX *d = reinterpret_cast<PX *>((plane ? cr : cb) + r.chroma_off) + blk_x(ke) + (size_t)blk_y(ke) * uvlsp;
        typename T::coef *b = gc + 16 * i;
        if (nz[scan8_of(e)]) T::idct4(bits, d, b, uvlsp); else if (b[0]) T::dc(bits, d, b, uvlsp, 4);
    }
}

// ---------------------------------------------------------------------------------------------------------------------------------
// clamped sample fetch = emulated_edge_mc (replicated borders); [y0, y0 + h) are the rows of the record's own picture
template <typename PX> struct EdgeFetchT {
    const PX *p; int st, w, h, y0;
    __device__ __forceinline__ int operator()(int x, int y) const { return p[(size_t)min(max(y, y0), y0 + h - 1) * st + min(max(x, 0), w - 1)]; }
};
// the (w + 5) x (h + 5) luma patch (or a (w / 2 + 1) x (ch + 1) chroma patch) of a partition staged in shared memory: sample (x, y) of the
// reference plane sits at p[(y - y0) * pitch + (x - x0)]
template <typename PX> struct PatchFetchT {
    const PX *p; int pitch, x0, y0;
    __device__ __forceinline__ int operator()(int x, int y) const { return p[(y - y0) * pitch + (x - x0)]; }
};
template <class F> __device__ __forceinline__ int tap6f(const F &S, int x, int y, int dx, int dy)
{ return (S(x, y) + S(x + dx, y + dy)) * 20 - (S(x - dx, y - dy) + S(x + 2 * dx, y + 2 * dy)) * 5 + (S(x - 2 * dx, y - 2 * dy) + S(x + 3 * dx, y + 3 * dy)); }
template <class F> __device__ __forceinline__ int qh(int bits, const F &S, int x, int y) { return hbd::clipb((tap6f(S, x, y, 1, 0) + 16) >> 5, bits); }
template <class F> __device__ __forceinline__ int qv(int bits, const F &S, int x, int y) { return hbd::clipb((tap6f(S, x, y, 0, 1) + 16) >> 5, bits); }
template <class F> __device__ inline int qhv(int bits, const F &S, int x, int y)
{
    int t[6];
    for (int k = 0; k < 6; k++) t[k] = tap6f(S, x, y + k - 2, 1, 0);
    return hbd::clipb(((t[2] + t[3]) * 20 - (t[1] + t[4]) * 5 + (t[0] + t[5]) + 512) >> 10, bits);
}
// the sixteen quarter-sample positions (h264qpel_template.c:380-531)
template <class F> __device__ inline int qpel_at(int bits, const F &S, int x, int y, int fx, int fy)
{
    int a, b = -1;
    if (!fx && !fy) a = S(x, y);
    else if (!fy) { a = qh(bits, S, x, y); if (fx != 2) b = S(x + (fx == 3), y); }
    else if (!fx) { a = qv(bits, S, x, y); if (fy != 2) b = S(x, y + (fy == 3)); }
    else if (fx == 2 && fy == 2) a = qhv(bits, S, x, y);
    else if (fx == 2) { a = qhv(bits, S, x, y); b = qh(bits, S, x, y + (fy == 3)); }
    else if (fy == 2) { a = qhv(bits, S, x, y); b = qv(bits, S, x + (fx == 3), y); }
    else { a = qh(bits, S, x, y + (fy == 3)); b = qv(bits, S, x + (fx == 3), y); }
    return b < 0 ? a : (a + b + 1) >> 1;
}
template <class F> __device__ __forceinline__ int chroma_at(const F &S, int x, int y, int A, int B, int Cc, int D)
{
    int v = A * S(x, y);
    if (B) v += B * S(x + 1, y);
    if (Cc) v += Cc * S(x, y + 1);
    if (D) v += D * S(x + 1, y + 1);
    return (v + 32) >> 6;
}

// STAGED: the warp first copies the clamped patches into its slice of shared memory (one global load per patch sample instead of 6 .. 36
// per output sample), then every lane filters from there.  !STAGED: every tap is a clamped global load -- the same arithmetic with no
// communication between lanes, which is what tests/hostsim/ compiles.
constexpr int MCH_LP = 24, MCH_CP = 12;           // patch pitches in samples (21 x 21 luma, 9 x 17 chroma per plane)
template <typename PX, bool STAGED>
__global__ void __launch_bounds__(128)
h264_mc_hbd_kernel(int bits, int c422, const FFH264MCRecord *__restrict__ recs, size_t n, const FFH264RefPlanes *__restrict__ refs,
                   uint8_t *__restrict__ dy, uint8_t *__restrict__ dcb, uint8_t *__restrict__ dcr, int ls, int uvls, int pw, int ph, int pass)
{
#ifndef AVB_HOSTSIM
    __shared__ PX s_luma[STAGED ? 4 : 1][STAGED ? 21 * MCH_LP : 1];
    __shared__ PX s_chroma[STAGED ? 4 : 1][2][STAGED ? 17 * MCH_CP : 1];
#endif
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const size_t ri = (size_t)blockIdx.x * 4 + warp;
    if (ri >= n) return;
    const FFH264MCRecord r = recs[ri];
    if ((r.avg != 0) != (pass != 0)) return;
    const FFH264RefPlanes ref = refs[r.ref];
    const int lsp = ls / (int)sizeof(PX), uvlsp = uvls / (int)sizeof(PX);
    const int ly0 = ((int)r.y / ph) * ph;                                   // first luma row of the record's picture in the stacked planes
    const int mx = (int)r.mvx + 4 * (int)r.x, my = (int)r.mvy + 4 * (int)r.y, w = r.w, h = r.h;
    // chroma: eighth-sample bilinear (h264chroma_template.c:27-173); 4:2:2 keeps the luma's vertical resolution (h264_mb.c:287-316)
    const int cw = w >> 1, ch = c422 ? h : h >> 1, cph = c422 ? ph : ph >> 1, cy0 = c422 ? ly0 : ly0 >> 1;
    const int sx = mx >> 3, sy = c422 ? my >> 2 : my >> 3, fx = mx & 7, fy = c422 ? (my << 1) & 7 : my & 7;
    const int dx0 = r.x >> 1, dy0 = c422 ? (int)r.y : r.y >> 1;
    const int A = (8 - fx) * (8 - fy), B = fx * (8 - fy), Cc = (8 - fx) * fy, D = fx * fy;
    const EdgeFetchT<PX> GY = { reinterpret_cast<const PX *>(ref.y), lsp, pw, ph, ly0 };
    PX *d0 = reinterpret_cast<PX *>(dy) + (size_t)r.y * lsp + r.x;
    (void)warp;
#ifndef AVB_HOSTSIM
    if (STAGED) {
        const int lx0 = (mx >> 2) - 2, lyy0 = (my >> 2) - 2;
        for (int i = lane; i < (w + 5) * (h + 5); i += 32) { const int c = i % (w + 5), rr = i / (w + 5); s_luma[warp][rr * MCH_LP + c] = (PX)GY(lx0 + c, lyy0 + rr); }
        for (int i = lane; i < 2 * (cw + 1) * (ch + 1); i += 32) {
            const int pl = i / ((cw + 1) * (ch + 1)), k = i % ((cw + 1) * (ch + 1)), c = k % (cw + 1), rr = k / (cw + 1);
            const EdgeFetchT<PX> GC = { reinterpret_cast<const PX *>(pl ? ref.cr : ref.cb), uvlsp, pw >> 1, cph, cy0 };
            s_chroma[warp][pl][rr * MCH_CP + c] = (PX)GC(sx + c, sy + rr);
        }
        __syncwarp();
        const PatchFetchT<PX> SY = { s_luma[warp], MCH_LP, lx0, lyy0 };
        for (int i = lane; i < w * h; i += 32) {
            const int x = i % w, y = i / w;
            const int v = qpel_at(bits, SY, (mx >> 2) + x, (my >> 2) + y, mx & 3, my & 3);
            PX *d = d0 + (size_t)y * lsp + x;
            *d = (PX)(r.avg ? (*d + v + 1) >> 1 : v);
        }
        for (int i = lane; i < 2 * cw * ch; i += 32) {
            const int pl = i / (cw * ch), k = i % (cw * ch), x = k % cw, y = k / cw;
            const PatchFetchT<PX> SC = { s_chroma[warp][pl], MCH_CP, sx, sy };
            const int v = chroma_at(SC, sx + x, sy + y, A, B, Cc, D);
            PX *d = reinterpret_cast<PX *>(pl ? dcr : dcb) + (size_t)(dy0 + y) * uvlsp + dx0 + x;
            *d = (PX)(r.avg ? (*d + v + 1) >> 1 : v);
        }
        return;
    }
#endif
    for (int i = lane; i < w * h; i += 32) {
        const int x = i % w, y = i / w;
        const int v = qpel_at(bits, GY, (mx >> 2) + x, (my >> 2) + y, mx & 3, my & 3);
        PX *d = d0 + (size_t)y * lsp + x;
        *d = (PX)(r.avg ? (*d + v + 1) >> 1 : v);
    }
    for (int i = lane; i < 2 * cw * ch; i += 32) {
        const int pl = i / (cw * ch), k = i % (cw * ch), x = k % cw, y = k / cw;
        const EdgeFetchT<PX> GC = { reinterpret_cast<const PX *>(pl ? ref.cr : ref.cb), uvlsp, pw >> 1, cph, cy0 };
        const int v = chroma_at(GC, sx + x, sy + y, A, B, Cc, D);
        PX *d = reinterpret_cast<PX *>(pl ? dcr : dcb) + (size_t)(dy0 + y) * uvlsp + dx0 + x;
        *d = (PX)(r.avg ? (*d + v + 1) >> 1 : v);
    }
}

// weight_h264_pixels / biweight_h264_pixels at 9 / 10 bit (h264dsp_template.c:30-98: the offset is scaled by 2^(bits - 8), :39,70): warp per record
__global__ void __launch_bounds__(128)
h264_weight_hbd_kernel(int bits, const FFH264WeightRecord *__restrict__ recs, size_t n, uint8_t *__restrict__ plane, const uint8_t *__restrict__ src, int stride)
{
    const int lane = threadIdx.x & 31;
    const size_t ri = (size_t)blockIdx.x * 4 + (threadIdx.x >> 5);
    if (ri >= n) return;
    const FFH264WeightRecord r = recs[ri];
    const int ld = r.log2_denom, sp = stride >> 1;
    int off = (int)r.offset * (1 << (bits - 8));
    if (!src) { off *= 1 << ld; if (ld) off += 1 << (ld - 1); }
    else off = ((off + 1) | 1) << ld;
    px *d0 = reinterpret_cast<px *>(plane + r.off);
    const px *s0 = src ? reinterpret_cast<const px *>(src + r.off) : nullptr;
    for (int it = lane; it < r.w * r.h; it += 32) {
        const size_t o = (size_t)(it / r.w) * sp + it % r.w;
        const int v = s0 ? ((int)s0[o] * r.weight_src + (int)d0[o] * r.weight + off) >> (ld + 1) : ((int)d0[o] * r.weight + off) >> ld;
        d0[o] = (px)hbd::clipb(v, bits);
    }
}

// h264_luma_dc_dequant_idct / h264_chroma_dc_dequant_idct / h264_chroma422_dc_dequant_idct on int32 coefficients (h264idct_template.c:242-324), the
// step hl_decode_mb() runs before the residual of a macroblock: thread per macroblock, only the DC positions of its arena are touched
__global__ void __launch_bounds__(128)
h264_dc_dequant_hbd_kernel(int c422, const FFH264DCRecord *__restrict__ recs, size_t n, int32_t *__restrict__ coeffs, size_t coeff_stride, const int32_t *__restrict__ luma_dc)
{
    const size_t m = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (m >= n) return;
    const FFH264DCRecord r = recs[m];
    int32_t *mb = coeffs + m * coeff_stride;
    if (r.luma_qmul) {
        int32_t in[16];
        for (int i = 0; i < 16; i++) in[i] = luma_dc[16 * m + i];
        hbd::luma_dc_dequant(mb, in, (int)r.luma_qmul);
    }
    for (int pl = 0; pl < 2; pl++)
        if (r.chroma_qmul[pl]) { if (c422) hbd::chroma422_dc_dequant(mb + 256 * (pl + 1), (int)r.chroma_qmul[pl]); else hbd::chroma_dc_dequant(mb + 256 * (pl + 1), (int)r.chroma_qmul[pl]); }
}

#ifndef AVB_HOSTSIM      // (the wavefront synchronises warps: not part of tests/hostsim/, GPU tests only)
// ---------------------------------------------------------------------------------------------------------------------------------
constexpr int DB_WARPS = 16;

__device__ __forceinline__ void prefetch_l1(const void *p) { asm volatile("prefetch.global.L1 [%0];" :: "l"(p)); }

// the loop-filter slots on one line across an edge, by sample type: 8-bit = h264dsp.cuh, 9 / 10-bit = h264dsp_hbd.cuh (alpha / beta / tc0
// scaled by 2^(bits - 8) like h264dsp_template.c:110-113,240); ctc = the chroma slots' tc0 argument (already + 1)
template <typename PX> struct LineFilter;
template <> struct LineFilter<uint8_t> {
    static __device__ __forceinline__ void luma(int, uint8_t *q, int ps, int a, int b, int tc0, bool intra)
    { if (intra) h264_luma_intra_line(q, ps, a, b); else if (tc0 >= 0) h264_luma_line(q, ps, a, b, tc0); }
    static __device__ __forceinline__ void chroma(int, uint8_t *q, int ps, int a, int b, int ctc, bool intra)
    { if (intra || ctc > 0) h264_chroma_line(q, ps, a, b, ctc, intra); }
};
template <> struct LineFilter<uint16_t> {
    static __device__ __forceinline__ void luma(int bits, uint16_t *q, int ps, int a, int b, int tc0, bool intra)
    { const int sh = bits - 8; if (intra) hbd::luma_intra_line(q, ps, a << sh, b << sh); else if (tc0 >= 0) hbd::luma_line(bits, q, ps, a << sh, b << sh, tc0 << sh); }
    static __device__ __forceinline__ void chroma(int bits, uint16_t *q, int ps, int a, int b, int ctc, bool intra)
    {
        const int sh = bits - 8;
        if (intra) hbd::chroma_line(bits, q, ps, a << sh, b << sh, 0, 1);
        else { const int tc = ((ctc - 1) << sh) + 1; if (tc > 0) hbd::chroma_line(bits, q, ps, a << sh, b << sh, tc, 0); }
    }
};

// blockIdx.x = picture, blockIdx.y = 0 luma / 1 chroma: the planes are independent (h264_loopfilter.c filters them edge by edge side by
// side, but no sample of one plane depends on another), so each gets its own CTA, its own wavefront and its own progress counters.
// Luma: lanes 0..15 = the 16 lines / columns of a macroblock.  Chroma 4:2:0: lanes 0..7 cb, 8..15 cr.  Chroma 4:2:2 (8 x 16 macroblocks):
// vertical edges = 16 lines per plane on all 32 lanes (two edges, the 104-byte record's fields, a tc0 entry per four lines), horizontal
// edges = 8 columns per plane on 16 lanes, FOUR edges (rows 0, 4, 8, 12; one per luma edge, h264_loopfilter.c:693-700) from the 52-byte
// FFH264DeblockChroma422 record.  While macroblock x is filtered the records and the sample rows of macroblock x + 1 are prefetched into
// L1 (first touches otherwise cost a DRAM round trip per macroblock on the critical path of the wavefront; the CTA is the only writer of
// its picture, so the SM's L1 stays coherent).
template <typename PX, bool C422>
__global__ void __launch_bounds__(DB_WARPS * 32)
h264_deblock_generic_kernel(int bits, const FFH264DeblockMB *__restrict__ mbs, const FFH264DeblockChroma422 *__restrict__ ext, int mb_w, int mb_h,
                            uint8_t *luma, uint8_t *cb, uint8_t *cr, int ls, int uvls)
{
    extern __shared__ int prog_s[];                                  // macroblocks finished per row of this CTA's picture and plane kind
    volatile int *prog = prog_s;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, pic = blockIdx.x;
    const bool is_luma = blockIdx.y == 0;
    for (int i = threadIdx.x; i < mb_h; i += blockDim.x) prog_s[i] = 0;
    __syncthreads();
    const int st = (is_luma ? ls : uvls) / (int)sizeof(PX);           // row distance in samples
    const int mbw_px = is_luma ? 16 : 8, mbh_px = is_luma ? 16 : (C422 ? 16 : 8);
    PX *const yplane = reinterpret_cast<PX *>(luma) + (size_t)pic * mb_h * 16 * st;
    PX *const cplane[2] = { reinterpret_cast<PX *>(cb) + (size_t)pic * mb_h * mbh_px * st, reinterpret_cast<PX *>(cr) + (size_t)pic * mb_h * mbh_px * st };
    // prefetch role of this lane: a sample row of the next macroblock (luma: rows 0..15 on lanes 0..15, the four rows above on 16..19;
    // chroma: plane lane >> 4, rows 0..mbh - 1, the two rows above on the lanes left over in 4:2:0)
    const int pf_plane = is_luma ? 0 : lane >> 4;
    int pf_row = is_luma ? (lane < 16 ? lane : lane < 20 ? 15 - lane : 99) : ((lane & 15) < mbh_px ? (lane & 15) : (lane & 15) < mbh_px + 2 ? mbh_px - 1 - (lane & 15) : 99);
    for (int row = warp; row < mb_h; row += DB_WARPS) {
        PX *const rbase_y = yplane + (size_t)row * 16 * st;
        PX *const rbase_c[2] = { cplane[0] + (size_t)row * mbh_px * st, cplane[1] + (size_t)row * mbh_px * st };
        PX *const pf_base = is_luma ? rbase_y : rbase_c[pf_plane];
        const size_t mrow = ((size_t)pic * mb_h + row) * mb_w;
        const bool pf_ok = pf_row != 99 && (pf_row >= 0 || row > 0);
        for (int x = -1; x < mb_w; x++) {
            if (x + 1 < mb_w) {                                       // macroblock x + 1: sample rows, the 104-byte record (4 sectors), the 52-byte one (2)
                if (pf_ok) prefetch_l1(pf_base + (ptrdiff_t)pf_row * st + (x + 1) * mbw_px);
                if (lane < 4) prefetch_l1(reinterpret_cast<const char *>(mbs + mrow + x + 1) + 32 * lane);
                else if (C422 && !is_luma && lane < 6) prefetch_l1(reinterpret_cast<const char *>(ext + mrow + x + 1) + 32 * (lane - 4));
            }
            if (x < 0) continue;
            if (row > 0) {
                // the row above must be done with macroblock x + 1: its left-edge filter still reads and writes columns 13..15 of the
                // macroblock above this one (raster order of the reference)
                const int need = min(x + 2, mb_w);
                if (lane == 0) while (prog[row - 1] < need) { }
                __syncwarp();
                __threadfence_block();
            }
            const FFH264DeblockMB &P = mbs[mrow + x];
            for (int dir = 0; dir < 2; dir++) {
                // dir 0: vertical edges, a lane = a line; dir 1: horizontal edges, a lane = a column
                if (is_luma) {
                    if (lane < 16) {
                        PX *const line = dir == 0 ? rbase_y + (size_t)lane * st + x * 16 : rbase_y + x * 16 + lane;
                        const int across = dir == 0 ? 1 : st;
                        for (int e = 0; e < 4; e++) {
                            const int a = P.alpha[dir][e], b = P.beta[dir][e];
                            if (a && b) LineFilter<PX>::luma(bits, line + (size_t)4 * e * across, across, a, b, P.tc0[dir][e][lane >> 2], P.intra[dir] >> e & 1);
                        }
                    }
                } else if (C422 && dir == 0) {
                    const int p = lane >> 4, l = lane & 15;                                 // 16 lines per plane
                    PX *const line = rbase_c[p] + (size_t)l * st + x * 8;
                    for (int e = 0; e < 2; e++) {
                        const int a = P.calpha[p][0][e], b = P.cbeta[p][0][e];
                        if (a && b) LineFilter<PX>::chroma(bits, line + 4 * e, 1, a, b, P.ctc0[p][0][e][l >> 2], P.cintra[p][0] >> e & 1);
                    }
                } else if (lane < 16) {
                    const int p = lane >> 3, l = lane & 7;
                    PX *const line = dir == 0 ? rbase_c[p] + (size_t)l * st + x * 8 : rbase_c[p] + x * 8 + l;
                    const int across = dir == 0 ? 1 : st;
                    if (C422) {                                                              // four horizontal edges from the 4:2:2 record
                        const FFH264DeblockChroma422 &X = ext[mrow + x];
                        for (int e = 0; e < 4; e++) {
                            const int a = X.alpha[p][e], b = X.beta[p][e];
                            if (a && b) LineFilter<PX>::chroma(bits, line + (size_t)4 * e * across, across, a, b, X.tc0[p][e][l >> 1], X.intra[p] >> e & 1);
                        }
                    } else {
                        for (int e = 0; e < 2; e++) {
                            const int a = P.calpha[p][dir][e], b = P.cbeta[p][dir][e];
                            if (a && b) LineFilter<PX>::chroma(bits, line + (size_t)4 * e * across, across, a, b, P.ctc0[p][dir][e][l >> 1], P.cintra[p][dir] >> e & 1);
                        }
                    }
                }
                __syncwarp();
                __threadfence_block();
            }
            if (lane == 0) prog[row] = x + 1;
        }
    }
}

// ---------------------------------------------------------------------------------------------------------------------------------
// Intra reconstruction at 9 / 10 bit, 4:2:0: hl_decode_mb() for the intra macroblocks of a batch of pictures (h264_mb.c:607-731 luma,
// h264_mb_template.c:158-197 chroma) -- per block pred4x4 / pred8x8l then its residual, pred16x16 then h264_idct_add16intra, pred8x8 on cb
// and cr then h264_idct_add8 -- in raster order.  One CTA per picture, its warps take macroblock rows round-robin as a wavefront two
// macroblocks behind the row above (prediction reaches left, up-left, up and up-right), progress in shared memory like the deblocking
// kernel above.  Every lane collects the block's neighbours itself (the table slots' PredJobH) and derives its samples from them;
// lane 0 (or a lane per 4x4 block) adds the residual; the warp synchronises between a block's prediction, its residual and the next block.
template <typename PX>
__device__ __forceinline__ void intra_job_neighbours(PredJobH &j, const PX *P, int st, int nt, int nl, bool tr_ok, int ax, int ay, int y0)
{   // P = the block's first sample at absolute (ax, ay); [y0, ..) = the picture's rows.  nt top samples (4 or 8 more when tr_ok), nl left samples
    const bool top = ay - 1 >= y0, left = ax - 1 >= 0;
    for (int k = 0; k < nt; k++) j.top[k] = top ? P[-st + k] : 0;
    for (int k = nt; k < 2 * nt && k < 16; k++) j.top[k] = (top && tr_ok) ? P[-st + k] : j.top[nt - 1];
    for (int k = 0; k < nl; k++) j.left[k] = left ? P[(ptrdiff_t)k * st - 1] : 0;
    j.corner = (top && left) ? P[-st - 1] : 0;
}

// PX = uint16_t: 9 / 10-bit pictures; uint8_t: the 8-bit 4:2:2 pictures (bits 8: the predictors below are the 8-bit formulas, DC_128 = 128, plane
// prediction clipped to 255).  C422: the chroma macroblock is 8 x 16 -- pred8x8[] holds the 8 x 16 predictors (h264pred.c:477-563) and the residual
// is h264_idct_add8_422 (h264idct_template.c:216-236).
template <typename PX, bool C422>
__global__ void __launch_bounds__(DB_WARPS * 32)
h264_intra_generic_kernel(int bits, const FFH264IntraMB *__restrict__ mbs, int mb_w, int mb_h, typename Transform<PX>::coef *__restrict__ coeffs, size_t coeff_stride,
                          const uint8_t *__restrict__ nnzc_all, uint8_t *luma, uint8_t *cb, uint8_t *cr, int ls, int uvls)
{
    typedef Transform<PX> T;
    typedef typename T::coef coef;
    extern __shared__ int prog_s[];
    volatile int *prog = prog_s;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, pic = blockIdx.x;
    for (int i = threadIdx.x; i < mb_h; i += blockDim.x) prog_s[i] = 0;
    __syncthreads();
    constexpr int CH = C422 ? 16 : 8;                                    // chroma rows per macroblock
    const int lsp = ls / (int)sizeof(PX), uvlsp = uvls / (int)sizeof(PX), y0 = pic * mb_h * 16, cy0 = pic * mb_h * CH;
    PX *const Y = reinterpret_cast<PX *>(luma), *const C2[2] = { reinterpret_cast<PX *>(cb), reinterpret_cast<PX *>(cr) };
    for (int row = warp; row < mb_h; row += DB_WARPS) {
        for (int x = 0; x < mb_w; x++) {
            const size_t m = ((size_t)pic * mb_h + row) * mb_w + x;
            const FFH264IntraMB M = mbs[m];
            if (M.kind) {
                if (row > 0) {
                    const int need = min(x + 2, mb_w);                 // up-right neighbour finished
                    if (lane == 0) while (prog[row - 1] < need) { }
                    __syncwarp();
                    __threadfence_block();
                }
                coef *mb = coeffs + m * coeff_stride;
                const uint8_t *nnzc = nnzc_all + m * 120;
                const int ax0 = x * 16, ay0 = y0 + row * 16;
                PredJobH j;
                j.bits = bits; j.has_tl = j.has_tr = 0; j.nblocks = 0;
                if (M.kind == 1) {                                      // intra 4x4: 16 blocks in coding order
                    for (int i = 0; i < 16; i++) {
                        const int bx = blk_x(i), by = blk_y(i), mode = M.mode4[i];
                        PX *P = Y + (size_t)(ay0 + by) * lsp + ax0 + bx;
                        const bool tr_ok = (M.topright_samples_available << i) & 0x8000;
                        j.tab = 0; j.mode = mode;
                        intra_job_neighbours(j, P, lsp, 4, 4, tr_ok, ax0 + bx, ay0 + by, y0);
                        int v = 0;
                        if (lane < 16) {
                            if (mode == 11) v = 1 << (bits - 1);
                            else { IntraEdges e; hbd_edges(e, j); v = intra_directional(e, 4, mode, lane & 3, lane >> 2); }
                        }
                        __syncwarp();                                   // every lane has read its neighbours
                        if (lane < 16) P[(size_t)(lane >> 2) * lsp + (lane & 3)] = (PX)v;
                        __syncwarp();
                        const int nnz = nnzc[scan8_of(i)];
                        if (lane == 0 && nnz) { if (nnz == 1 && mb[16 * i]) T::dc(bits, P, mb + 16 * i, lsp, 4); else T::idct4(bits, P, mb + 16 * i, lsp); }
                        __syncwarp();
                    }
                } else if (M.kind == 2) {                               // intra 8x8 (pred8x8l)
                    for (int k = 0; k < 4; k++) {
                        const int i = 4 * k, bx = 8 * (k & 1), by = 8 * (k >> 1), mode = M.mode4[i];
                        PX *P = Y + (size_t)(ay0 + by) * lsp + ax0 + bx;
                        j.tab = 1; j.mode = mode;
                        j.has_tl = ((M.topleft_samples_available << i) & 0x8000) != 0; j.has_tr = ((M.topright_samples_available << i) & 0x4000) != 0;
                        intra_job_neighbours(j, P, lsp, 8, 8, j.has_tr, ax0 + bx, ay0 + by, y0);
                        int v[2];
                        {
                            IntraEdges e;
                            if (mode != 11) hbd_edges(e, j);
                            for (int q = 0; q < 2; q++) { const int sidx = lane + 32 * q; v[q] = mode == 11 ? 1 << (bits - 1) : intra_directional(e, 8, mode, sidx & 7, sidx >> 3); }
                        }
                        __syncwarp();
                        for (int q = 0; q < 2; q++) { const int sidx = lane + 32 * q; P[(size_t)(sidx >> 3) * lsp + (sidx & 7)] = (PX)v[q]; }
                        __syncwarp();
                        const int nnz = nnzc[scan8_of(i)];
                        if (lane == 0 && nnz) { if (nnz == 1 && mb[16 * i]) T::dc(bits, P, mb + 16 * i, lsp, 8); else T::idct8(bits, P, mb + 16 * i, lsp); }
                        __syncwarp();
                    }
                    j.has_tl = j.has_tr = 0;
                } else {                                                // intra 16x16, then h264_idct_add16intra
                    PX *P = Y + (size_t)ay0 * lsp + ax0;
                    j.tab = 3; j.mode = M.mode16;
                    intra_job_neighbours(j, P, lsp, 16, 16, false, ax0, ay0, y0);
                    int v[8];
                    for (int q = 0; q < 8; q++) { const int sidx = lane + 32 * q; v[q] = hbd_big_sample(j, 16, sidx & 15, sidx >> 4); }
                    __syncwarp();
                    for (int q = 0; q < 8; q++) { const int sidx = lane + 32 * q; P[(size_t)(sidx >> 4) * lsp + (sidx & 15)] = (PX)v[q]; }
                    __syncwarp();
                    if (lane < 16) {
                        PX *d = P + (size_t)blk_y(lane) * lsp + blk_x(lane);
                        if (nnzc[scan8_of(lane)]) T::idct4(bits, d, mb + 16 * lane, lsp); else if (mb[16 * lane]) T::dc(bits, d, mb + 16 * lane, lsp, 4);
                    }
                    __syncwarp();
                }
                // chroma: pred8x8 on both planes, then h264_idct_add8 (4:2:2: the 8 x 16 predictors, then h264_idct_add8_422)
                const int crow = cy0 + row * CH;
                for (int pl = 0; pl < 2; pl++) {
                    PX *P = C2[pl] + (size_t)crow * uvlsp + x * 8;
                    j.tab = C422 ? 5 : 2; j.mode = M.chroma_mode;
                    intra_job_neighbours(j, P, uvlsp, 8, CH, false, x * 8, crow, cy0);
                    int v[CH / 4];
                    for (int q = 0; q < CH / 4; q++) { const int sidx = lane + 32 * q; v[q] = C422 ? hbd_sample_8x16(j, sidx & 7, sidx >> 3) : hbd_big_sample(j, 8, sidx & 7, sidx >> 3); }
                    __syncwarp();
                    for (int q = 0; q < CH / 4; q++) { const int sidx = lane + 32 * q; P[(size_t)(sidx >> 3) * uvlsp + (sidx & 7)] = (PX)v[q]; }
                }
                __syncwarp();
                constexpr int PER = C422 ? 8 : 4;                        // 4x4 chroma blocks per plane
                if (M.chroma_residual && lane < 2 * PER) {
                    // 4:2:2: the lower four blocks keep their coefficients at block i but are addressed through scan8[i + 4] (rows 8..15)
                    const int pl = lane / PER, k = lane % PER, i = 16 + 16 * pl + k, e = k >= 4 ? i + 4 : i, ke = e & 15;
                    PX *d = C2[pl] + (size_t)(crow + blk_y(ke)) * uvlsp + x * 8 + blk_x(ke);
                    if (nnzc[scan8_of(e)]) T::idct4(bits, d, mb + 16 * i, uvlsp); else if (mb[16 * i]) T::dc(bits, d, mb + 16 * i, uvlsp, 4);
                }
                __syncwarp();
                __threadfence_block();
            }
            if (lane == 0) prog[row] = x + 1;
        }
    }
}

#endif

bool hbd_args_ok(const char *where, int bit_depth, int chroma_format_idc, int ls, int uvls, const void *a, const void *b, const void *c)
{
    if (bit_depth != 9 && bit_depth != 10) { set_error_msg(where, "bit_depth must be 9 or 10 (8-bit pictures take the calls without _hbd)"); return false; }
    if (chroma_format_idc != 1 && chroma_format_idc != 2) { set_error_msg(where, "chroma_format_idc must be 1 (4:2:0) or 2 (4:2:2)"); return false; }
    if (((uintptr_t)a | (uintptr_t)b | (uintptr_t)c | (uintptr_t)ls | (uintptr_t)uvls) & 1) { set_error_msg(where, "16-bit samples need even plane addresses and pitches"); return false; }
    return true;
}

// bit_depth 8 is taken for chroma_format_idc 2 only (8-bit 4:2:0 has the kernels of h264_residual.cu / h264_mc.cu behind the calls without _hbd)
static bool depth_idc_ok(const char *where, int bit_depth, int chroma_format_idc, int ls, int uvls, const void *a, const void *b, const void *c)
{
    if (bit_depth == 8) {
        if (chroma_format_idc != 2) { set_error_msg(where, "bit_depth 8 is taken with chroma_format_idc 2 only (8-bit 4:2:0: the calls without _hbd)"); return false; }
        return true;
    }
    return hbd_args_ok(where, bit_depth, chroma_format_idc, ls, uvls, a, b, c);
}

template <typename PX>
static int launch_mc_generic(int bit_depth, int c422, const FFH264MCRecord *recs, size_t n, const FFH264RefPlanes *refs, uint8_t *dst_y, uint8_t *dst_cb, uint8_t *dst_cr,
                             int linesize, int uvlinesize, int pic_w, int pic_h, cudaStream_t st)
{
    for (int pass = 0; pass < 2; pass++) {
#ifdef AVB_HOSTSIM
        AVB_LAUNCH((h264_mc_hbd_kernel<PX, false>), dim3((unsigned)((n + 3) / 4)), dim3(128), 0, st)(bit_depth, c422, recs, n, refs, dst_y, dst_cb, dst_cr, linesize, uvlinesize, pic_w, pic_h, pass);
#else
        if (tuning("mc_hbd_staged") == 2)       // (test knob: the clamped-global-load form of the same arithmetic, the one tests/hostsim/ runs)
            h264_mc_hbd_kernel<PX, false><<<(unsigned)((n + 3) / 4), 128, 0, st>>>(bit_depth, c422, recs, n, refs, dst_y, dst_cb, dst_cr, linesize, uvlinesize, pic_w, pic_h, pass);
        else
            h264_mc_hbd_kernel<PX, true><<<(unsigned)((n + 3) / 4), 128, 0, st>>>(bit_depth, c422, recs, n, refs, dst_y, dst_cb, dst_cr, linesize, uvlinesize, pic_w, pic_h, pass);
#endif
    }
    return 0;
}

#ifndef AVB_HOSTSIM
template <typename PX, bool C422>
static int launch_intra_generic(const char *where, int bit_depth, const FFH264IntraMB *mbs, int mb_w, int mb_h, int n_pictures, void *coeffs, size_t coeff_stride,
                                const uint8_t *nnzc, uint8_t *luma, uint8_t *cb, uint8_t *cr, int ls, int uvls, cudaStream_t st)
{
    if (!mbs || !coeffs || !nnzc || !luma || !cb || !cr || mb_w <= 0 || mb_h <= 0 || n_pictures < 0 || mb_h > 8192) { set_error_msg(where, "bad argument"); return -1; }
    if ((uintptr_t)coeffs % sizeof(typename Transform<PX>::coef)) { set_error_msg(where, "coeffs must be aligned to its coefficient type (int16 at 8 bit, int32 at 9 / 10)"); return -1; }
    if (!n_pictures) return 0;
    h264_intra_generic_kernel<PX, C422><<<(unsigned)n_pictures, DB_WARPS * 32, (size_t)mb_h * sizeof(int), st>>>(
        bit_depth, mbs, mb_w, mb_h, static_cast<typename Transform<PX>::coef *>(coeffs), coeff_stride, nnzc, luma, cb, cr, ls, uvls);
    return check_launch(where) ? -1 : 0;
}
#endif

}  // namespace
}  // namespace avb

using namespace avb;

extern "C" {

int ff_h264_idct_add_mb_batch_hbd_cuda(int bit_depth, int chroma_format_idc, const FFH264ResidualMB *mbs, size_t n, int32_t *coeffs, size_t coeff_stride,
                                       const uint8_t *nnzc, uint8_t *luma, uint8_t *cb, uint8_t *cr, int linesize, int uvlinesize, void *stream)
{
    avb::enter();
    const char *where = "ff_h264_idct_add_mb_batch_hbd_cuda";
    if (!depth_idc_ok(where, bit_depth, chroma_format_idc, linesize, uvlinesize, luma, cb, cr)) return -1;
    if (n && (!mbs || !coeffs || !nnzc || !luma || !cb || !cr)) { set_error_msg(where, "NULL argument"); return -1; }
    if (!n) return 0;
    if (bit_depth == 8)         // int16 coefficients behind the pointer
        AVB_LAUNCH(h264_residual_hbd_kernel<uint8_t>, dim3((unsigned)((n + 3) / 4)), dim3(128), 0, (cudaStream_t)stream)(8, 1, mbs, n, (int16_t *)coeffs, coeff_stride, nnzc,
                                                                                                                         luma, cb, cr, linesize, uvlinesize);
    else
        AVB_LAUNCH(h264_residual_hbd_kernel<uint16_t>, dim3((unsigned)((n + 3) / 4)), dim3(128), 0, (cudaStream_t)stream)(bit_depth, chroma_format_idc == 2, mbs, n, coeffs, coeff_stride, nnzc,
                                                                                                                          luma, cb, cr, linesize, uvlinesize);
    return check_launch(where) ? -1 : 0;
}

int ff_h264_mc_batch_hbd_cuda(int bit_depth, int chroma_format_idc, const FFH264MCRecord *recs, size_t n, const FFH264RefPlanes *refs, uint8_t *dst_y,
                              uint8_t *dst_cb, uint8_t *dst_cr, int linesize, int uvlinesize, int pic_w, int pic_h, void *stream)
{
    avb::enter();
    const char *where = "ff_h264_mc_batch_hbd_cuda";
    if (!depth_idc_ok(where, bit_depth, chroma_format_idc, linesize, uvlinesize, dst_y, dst_cb, dst_cr)) return -1;
    if (n && (!recs || !refs || !dst_y || !dst_cb || !dst_cr)) { set_error_msg(where, "NULL argument"); return -1; }
    if (pic_w <= 0 || pic_h <= 0 || (pic_w & 1) || (pic_h & 1)) { set_error_msg(where, "picture size must be positive and even"); return -1; }
    if (!n) return 0;
    if (bit_depth == 8) launch_mc_generic<uint8_t>(8, 1, recs, n, refs, dst_y, dst_cb, dst_cr, linesize, uvlinesize, pic_w, pic_h, (cudaStream_t)stream);
    else launch_mc_generic<uint16_t>(bit_depth, chroma_format_idc == 2, recs, n, refs, dst_y, dst_cb, dst_cr, linesize, uvlinesize, pic_w, pic_h, (cudaStream_t)stream);
    return check_launch(where) ? -1 : 0;
}

int ff_h264_weight_batch_hbd_cuda(int bit_depth, const FFH264WeightRecord *recs, size_t n, uint8_t *plane, const uint8_t *src, int stride, void *stream)
{
    avb::enter();
    const char *where = "ff_h264_weight_batch_hbd_cuda";
    if (!hbd_args_ok(where, bit_depth, 1, stride, 0, plane, src, nullptr)) return -1;
    if (n && (!recs || !plane)) { set_error_msg(where, "NULL argument"); return -1; }
    if (!n) return 0;
    AVB_LAUNCH(h264_weight_hbd_kernel, dim3((unsigned)((n + 3) / 4)), dim3(128), 0, (cudaStream_t)stream)(bit_depth, recs, n, plane, src, stride);
    return check_launch(where) ? -1 : 0;
}

int ff_h264_dc_dequant_batch_hbd_cuda(int chroma_format_idc, const FFH264DCRecord *recs, size_t n, int32_t *coeffs, size_t coeff_stride, const int32_t *luma_dc, void *stream)
{
    avb::enter();
    const char *where = "ff_h264_dc_dequant_batch_hbd_cuda";
    if (chroma_format_idc != 1 && chroma_format_idc != 2) { set_error_msg(where, "chroma_format_idc must be 1 or 2"); return -1; }
    if (n && (!recs || !coeffs || !luma_dc)) { set_error_msg(where, "NULL argument"); return -1; }
    if (!n) return 0;
    AVB_LAUNCH(h264_dc_dequant_hbd_kernel, dim3((unsigned)((n + 127) / 128)), dim3(128), 0, (cudaStream_t)stream)(chroma_format_idc == 2, recs, n, coeffs, coeff_stride, luma_dc);
    return check_launch(where) ? -1 : 0;
}

#ifndef AVB_HOSTSIM
int ff_h264_intra_mb_batch_hbd_cuda(int bit_depth, const FFH264IntraMB *mbs, int mb_w, int mb_h, int n_pictures, int32_t *coeffs, size_t coeff_stride,
                                    const uint8_t *nnzc, uint8_t *luma, uint8_t *cb, uint8_t *cr, int linesize, int uvlinesize, void *stream)
{
    avb::enter();
    const char *where = "ff_h264_intra_mb_batch_hbd_cuda";
    if (!hbd_args_ok(where, bit_depth, 1, linesize, uvlinesize, luma, cb, cr)) return -1;
    return launch_intra_generic<uint16_t, false>(where, bit_depth, mbs, mb_w, mb_h, n_pictures, coeffs, coeff_stride, nnzc, luma, cb, cr, linesize, uvlinesize, (cudaStream_t)stream);
}

int ff_h264_intra_mb_batch_422_cuda(int bit_depth, const FFH264IntraMB *mbs, int mb_w, int mb_h, int n_pictures, void *coeffs, size_t coeff_stride,
                                    const uint8_t *nnzc, uint8_t *luma, uint8_t *cb, uint8_t *cr, int linesize, int uvlinesize, void *stream)
{
    avb::enter();
    const char *where = "ff_h264_intra_mb_batch_422_cuda";
    if (!depth_idc_ok(where, bit_depth, 2, linesize, uvlinesize, luma, cb, cr)) return -1;
    if (bit_depth == 8)
        return launch_intra_generic<uint8_t, true>(where, 8, mbs, mb_w, mb_h, n_pictures, coeffs, coeff_stride, nnzc, luma, cb, cr, linesize, uvlinesize, (cudaStream_t)stream);
    return launch_intra_generic<uint16_t, true>(where, bit_depth, mbs, mb_w, mb_h, n_pictures, coeffs, coeff_stride, nnzc, luma, cb, cr, linesize, uvlinesize, (cudaStream_t)stream);
}
#endif

#ifndef AVB_HOSTSIM
static int launch_deblock_generic(const char *where, int bit_depth, const FFH264DeblockMB *mbs, const FFH264DeblockChroma422 *ext, int mb_w, int mb_h, int n_pictures,
                                  uint8_t *luma, uint8_t *cb, uint8_t *cr, int ls, int uvls, cudaStream_t st)
{
    if (!mbs || !luma || !cb || !cr || mb_w <= 0 || mb_h <= 0 || n_pictures < 0 || mb_h > 8192) { set_error_msg(where, "bad argument"); return -1; }
    if (!n_pictures) return 0;
    const dim3 grid((unsigned)n_pictures, 2);
    const size_t smem = (size_t)mb_h * sizeof(int);
    if (bit_depth == 8) {
        if (ext) h264_deblock_generic_kernel<uint8_t, true><<<grid, DB_WARPS * 32, smem, st>>>(8, mbs, ext, mb_w, mb_h, luma, cb, cr, ls, uvls);
        else     h264_deblock_generic_kernel<uint8_t, false><<<grid, DB_WARPS * 32, smem, st>>>(8, mbs, ext, mb_w, mb_h, luma, cb, cr, ls, uvls);
    } else {
        if (ext) h264_deblock_generic_kernel<uint16_t, true><<<grid, DB_WARPS * 32, smem, st>>>(bit_depth, mbs, ext, mb_w, mb_h, luma, cb, cr, ls, uvls);
        else     h264_deblock_generic_kernel<uint16_t, false><<<grid, DB_WARPS * 32, smem, st>>>(bit_depth, mbs, ext, mb_w, mb_h, luma, cb, cr, ls, uvls);
    }
    return check_launch(where) ? -1 : 0;
}

int ff_h264_deblock_batch_hbd_cuda(int bit_depth, const FFH264DeblockMB *mbs, int mb_w, int mb_h, int n_pictures, uint8_t *luma, uint8_t *cb, uint8_t *cr,
                                   int linesize, int uvlinesize, void *stream)
{
    avb::enter();
    const char *where = "ff_h264_deblock_batch_hbd_cuda";
    if (!hbd_args_ok(where, bit_depth, 1, linesize, uvlinesize, luma, cb, cr)) return -1;
    return launch_deblock_generic(where, bit_depth, mbs, nullptr, mb_w, mb_h, n_pictures, luma, cb, cr, linesize, uvlinesize, (cudaStream_t)stream);
}

int ff_h264_deblock_batch_422_cuda(int bit_depth, const FFH264DeblockMB *mbs, const FFH264DeblockChroma422 *chroma422, int mb_w, int mb_h, int n_pictures,
                                   uint8_t *luma, uint8_t *cb, uint8_t *cr, int linesize, int uvlinesize, void *stream)
{
    avb::enter();
    const char *where = "ff_h264_deblock_batch_422_cuda";
    if (bit_depth != 8 && !hbd_args_ok(where, bit_depth, 2, linesize, uvlinesize, luma, cb, cr)) return -1;
    if (!chroma422) { set_error_msg(where, "the 4:2:2 records are NULL"); return -1; }
    return launch_deblock_generic(where, bit_depth, mbs, chroma422, mb_w, mb_h, n_pictures, luma, cb, cr, linesize, uvlinesize, (cudaStream_t)stream);
}
#endif

}  // extern "C"
