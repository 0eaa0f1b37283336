// libav_b200/csrc/me_cmp.cu -- MECmpContext metrics, exhaustive motion search, HpelDSPContext and FDCTDSPContext
// batches for sm_90a.  Bit-exact replacements of
//   pix_abs / sad / sse / hadamard8_diff / hadamard8_intra / vsad / vsse / nsse / sum_abs_dctelem
//                                                      libavcodec/me_cmp.c:29-357, :434-536, :784-885
//   full_search + get_limits (restricted MVs, lambda 0) libavcodec/motion_est_template.c:620-655, motion_est.c:517-548
//   put / avg / no_rnd half-pel MC                      libavcodec/hpeldsp.c:38-366
//   jpeg_fdct_islow_8, fdct248_islow_8, fdct_ifast(248) libavcodec/jfdctint_template.c:182-398, jfdctfst.c:141-332
// Compare metrics: one warp per (block pair) record, lanes stride over samples, warp-shuffle reduction tree;
// the 8x8 Hadamard runs 8 lanes per block (lane = row) with the column butterflies done by __shfl_xor.
// Full search: one CTA per macroblock, 48x48 reference window staged in shared memory, current block in
// registers, 4-byte SAD (vabsdiff4) per word, candidates flattened in raster order so that the packed key
// (sad << 11 | raster index) reproduces the reference's strict-< first-wins tie break.
#include "common.cuh"
#include "fdct_dev.cuh"
#include "../../include/avdsp_b200.h"

namespace avb { int fdct10_launch(int which, int16_t *blocks, size_t n, cudaStream_t st); }      // fdct10.cu
namespace avb { int faan_fdct_launch(int which, int16_t *blocks, size_t n, cudaStream_t st); }   // faan_idct.cu

namespace avb {

__device__ __forceinline__ int iabs_m(int v) { return v < 0 ? -v : v; }
__device__ __forceinline__ int warp_sum(int v)
{
#pragma unroll
    for (int o = 16; o; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}

// ---- 8x8 Hadamard on 8 consecutive lanes (lane & 7 = row); returns the block's sum of |coeff| in every lane ----
__device__ __forceinline__ int hadamard8_lanes(const uint8_t *a, const uint8_t *b, ptrdiff_t st, int intra, int lane)
{
    const int row = lane & 7;
    int v[8];
#pragma unroll
    for (int x = 0; x < 8; x++) v[x] = intra ? a[row * st + x] : (int)b[row * st + x] - (int)a[row * st + x];
#pragma unroll
    for (int len = 1; len < 8; len <<= 1)                    // row transform in registers
#pragma unroll
        for (int i = 0; i < 8; i++)
            if (!(i & len)) { int p = v[i], q = v[i + len]; v[i] = p + q; v[i + len] = p - q; }
#pragma unroll
    for (int len = 1; len < 8; len <<= 1)                    // column transform across the 8 lanes
#pragma unroll
        for (int x = 0; x < 8; x++) {
            int o = __shfl_xor_sync(0xffffffffu, v[x], len);
            v[x] = (row & len) ? o - v[x] : v[x] + o;
        }
    int s = 0;
#pragma unroll
    for (int x = 0; x < 8; x++) s += iabs_m(v[x]);
    if (intra && row == 0) s -= iabs_m(v[0]);                // minus the mean (me_cmp.c:533)
    s += __shfl_xor_sync(0xffffffffu, s, 1);
    s += __shfl_xor_sync(0xffffffffu, s, 2);
    s += __shfl_xor_sync(0xffffffffu, s, 4);
    return s;
}

__global__ void __launch_bounds__(128)
me_cmp_kernel(int kind, int sidx, int dxy, const uint8_t *__restrict__ cur, const uint8_t *__restrict__ ref, ptrdiff_t st, int h,
              const FFMECmpRecord *__restrict__ recs, size_t n, int32_t *__restrict__ out)
{
    const int lane = threadIdx.x & 31;
    size_t ri = (size_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    if (ri >= n) return;
    const uint8_t *a = cur + recs[ri].cur_off, *b = ref + recs[ri].ref_off;
    const int w = sidx == 0 ? 16 : sidx == 1 ? 8 : 4;
    int s = 0;
    if (kind == 3 || kind == 7) {                            // hadamard8_diff / hadamard8_intra (+ 16-wide wrappers :859-874)
        const int intra = kind == 7, nblk = sidx == 0 ? (h == 16 ? 4 : 2) : 1, blk = lane >> 3;
        const int eb = blk < nblk ? blk : 0;                 // idle lanes recompute block 0 (they still take part in the shuffles)
        const int bx = (eb & 1) * 8, by = (eb >> 1) * 8;
        int v = hadamard8_lanes(a + by * st + bx, b + by * st + bx, st, intra, lane);   // all lanes participate in the shuffles
        s = (blk < nblk && (lane & 7) == 0) ? v : 0;
        s = warp_sum(s);
    } else if (kind == 10) {                                 // sum_abs_dctelem
        const int16_t *c = reinterpret_cast<const int16_t *>(a);
        s = warp_sum(iabs_m(c[lane]) + iabs_m(c[lane + 32]));
    } else {
        int s2 = 0;
        for (int it = lane; it < w * h; it += 32) {
            const int x = it % w, y = it / w;
            const uint8_t *p = a + y * st + x, *q = b + y * st + x;
            switch (kind) {
            case 0: case 1: {
                int d = kind == 1 ? 0 : dxy;
                int r = d == 0 ? q[0] : d == 1 ? (q[0] + q[1] + 1) >> 1 : d == 2 ? (q[0] + q[st] + 1) >> 1 : (q[0] + q[1] + q[st] + q[st + 1] + 2) >> 2;
                s += iabs_m(p[0] - r);
            } break;
            case 2: { int d = p[0] - q[0]; s += d * d; } break;
            case 4: case 5: if (y > 0) { int d = p[-st] - q[-st] - p[0] + q[0]; s += kind == 4 ? iabs_m(d) : d * d; } break;
            case 8: case 9: if (y > 0) { int d = p[-st] - p[0]; s += kind == 8 ? iabs_m(d) : d * d; } break;
            case 6: {
                int d = p[0] - q[0]; s += d * d;
                if (y + 1 < h && x + 1 < w) s2 += iabs_m(p[0] - p[st] - p[1] + p[st + 1]) - iabs_m(q[0] - q[st] - q[1] + q[st + 1]);
            } break;
            }
        }
        s = warp_sum(s);
        if (kind == 6) s += iabs_m(warp_sum(s2)) * 8;        // nsse weight 8 = the NULL-context default (me_cmp.c:331)
    }
    if (lane == 0) out[ri] = s;
}

// ---------------------------------------------------------------------------------------------------
constexpr int FS_R = 16, FS_WIN = 48, FS_PITCH = 52;          // search range, window edge, smem pitch (words: 13)

// ---------------------------------------------------------------------------------------------------
// Full search, register-tiled.  The 48x52 window is stored four times in shared memory, copy s shifted
// left by s bytes, so every candidate reads ALIGNED words (no funnel shifts), and a thread owns five vertically adjacent
// candidates of one column: the 20 reference rows it needs are read once (80 LDS.32) and reused by up to five
// candidates, 320 vabsdiff4 per thread.  33 columns x 7 row groups = 231 of the 256 threads carry work.  Copies are
// spaced 8 banks apart, which makes the 32 lanes of a warp (consecutive dx) hit 32 different banks.
constexpr int FS2_ROWW = 12;                                   // words per window row in a shifted copy (48 bytes)
constexpr int FS2_ROWS = FS_WIN + 2;                            // two spare rows: the last row group reads past the window (those candidates are invalid)
constexpr int FS2_COPY = FS2_ROWS * FS2_ROWW + 16;             // words per copy; 616 = 8 (mod 32): consecutive copies sit 8 banks apart
static_assert(FS2_COPY % 32 == 8, "the four shifted copies must start 8 banks apart");
constexpr int FS2_DYG = 5;

__global__ void __launch_bounds__(256)
full_search_kernel_v2(const uint8_t *__restrict__ cur, const uint8_t *__restrict__ ref, int stride, int w, int h, int mb_y0,
                      int32_t *__restrict__ out)
{
    __shared__ __align__(16) uint32_t raw[FS_WIN * 13];        // 52 bytes per row
    __shared__ __align__(16) uint32_t win[4 * FS2_COPY];
    __shared__ unsigned long long best_s[8];
    const int mbw = w >> 4, mbx = blockIdx.x, mby = mb_y0 + blockIdx.y, t = threadIdx.x;
    const int px = mbx * 16, py = mby * 16;
    // A window that lies inside the picture (all but the border macroblocks) is fetched as aligned words, and the four
    // byte-shifted copies are produced straight from the two words a thread loaded (no staging pass, one barrier).
    const bool interior = px >= FS_R && px + 36 <= w && py >= FS_R && py + 32 <= h && !((stride | (int)(uintptr_t)ref) & 3);
    if (interior) {
        const uint8_t *g = ref + (size_t)(py - FS_R) * stride + px - FS_R;
        for (int i = t; i < FS_WIN * FS2_ROWW; i += 256) {
            const int r = i / FS2_ROWW, cw = i - r * FS2_ROWW;
            const uint32_t *gp = reinterpret_cast<const uint32_t *>(g + (size_t)r * stride) + cw;
            const uint32_t a = __ldg(gp), b = __ldg(gp + 1);
            win[i] = a;
            win[FS2_COPY + i] = __funnelshift_r(a, b, 8);
            win[2 * FS2_COPY + i] = __funnelshift_r(a, b, 16);
            win[3 * FS2_COPY + i] = __funnelshift_r(a, b, 24);
        }
    } else {
        for (int i = t; i < FS_WIN * 13; i += 256) {
            const int r = i / 13, c4 = i % 13, gy = min(max(py - FS_R + r, 0), h - 1);
            uint32_t v = 0;
#pragma unroll
            for (int k = 0; k < 4; k++) v |= (uint32_t)__ldg(ref + (size_t)gy * stride + min(max(px - FS_R + 4 * c4 + k, 0), w - 1)) << (8 * k);
            raw[i] = v;
        }
        __syncthreads();
        for (int i = t; i < 4 * FS_WIN * FS2_ROWW; i += 256) {
            const int s = i / (FS_WIN * FS2_ROWW), rem = i % (FS_WIN * FS2_ROWW), r = rem / FS2_ROWW, cw = rem % FS2_ROWW;
            win[s * FS2_COPY + rem] = __funnelshift_r(raw[r * 13 + cw], raw[r * 13 + cw + 1], 8 * s);
        }
    }
    uint32_t c[16][4];
#pragma unroll
    for (int r = 0; r < 16; r++) {
        const uint4 v = *reinterpret_cast<const uint4 *>(cur + (size_t)(py + r) * stride + px);
        c[r][0] = v.x; c[r][1] = v.y; c[r][2] = v.z; c[r][3] = v.w;
    }
    __syncthreads();

    const int xmin = max(-px, -FS_R), xmax = min(w - 16 - px, FS_R), ymin = max(-py, -FS_R), ymax = min(h - 16 - py, FS_R);
    unsigned long long best = ~0ull;
    if (t < 33 * 7) {
        const int dxi = t % 33, g = t / 33, dy0 = g * FS2_DYG;                      // candidates (dxi, dy0 .. dy0 + 4), biased by +16
        const uint32_t *base = &win[(dxi & 3) * FS2_COPY + (dxi >> 2)];
        unsigned sad[FS2_DYG] = { 0, 0, 0, 0, 0 };
#pragma unroll
        for (int rr = 0; rr < 16 + FS2_DYG - 1; rr++) {
            const uint32_t *row = base + (dy0 + rr) * FS2_ROWW;                      // rows 48, 49 (spare) only feed invalid candidates
            const uint32_t w0 = row[0], w1 = row[1], w2 = row[2], w3 = row[3];
#pragma unroll
            for (int j = 0; j < FS2_DYG; j++) {
                const int cr = rr - j;
                if (cr >= 0 && cr < 16) {
                    // the accumulate is part of the instruction (VABSDIFF4 ... .ADD); written as `__vsadu4() + acc` the compiler
                    // split half of them into a separate IADD3 on the same (ALU) pipe
                    asm("vabsdiff4.u32.u32.u32.add %0, %1, %2, %0;" : "+r"(sad[j]) : "r"(c[cr][0]), "r"(w0));
                    asm("vabsdiff4.u32.u32.u32.add %0, %1, %2, %0;" : "+r"(sad[j]) : "r"(c[cr][1]), "r"(w1));
                    asm("vabsdiff4.u32.u32.u32.add %0, %1, %2, %0;" : "+r"(sad[j]) : "r"(c[cr][2]), "r"(w2));
                    asm("vabsdiff4.u32.u32.u32.add %0, %1, %2, %0;" : "+r"(sad[j]) : "r"(c[cr][3]), "r"(w3));
                }
            }
        }
        const int dx = dxi - FS_R;
#pragma unroll
        for (int j = 0; j < FS2_DYG; j++) {
            const int dy = dy0 + j - FS_R;
            if (dx >= xmin && dx <= xmax && dy >= ymin && dy <= ymax) {
                const unsigned long long key = ((unsigned long long)sad[j] << 11) | (unsigned)((dy0 + j) * 33 + dxi);
                best = key < best ? key : best;
            }
        }
    }
#pragma unroll
    for (int o = 16; o; o >>= 1) { unsigned long long v = __shfl_xor_sync(0xffffffffu, best, o); best = v < best ? v : best; }
    if ((t & 31) == 0) best_s[t >> 5] = best;
    __syncthreads();
    if (t == 0) {
#pragma unroll
        for (int k = 1; k < 8; k++) best = best_s[k] < best ? best_s[k] : best;
        const int idx = (int)(best & 2047);
        int32_t *o = out + 3 * ((size_t)mby * mbw + mbx);
        o[0] = idx % 33 - FS_R; o[1] = idx / 33 - FS_R; o[2] = (int32_t)(best >> 11);
    }
}

// ---------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(128)
hpel_kernel(const FFHpelRecord *__restrict__ recs, size_t n, uint8_t *__restrict__ dst, const uint8_t *__restrict__ src, ptrdiff_t st)
{
    const int lane = threadIdx.x & 31;
    size_t ri = (size_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    if (ri >= n) return;
    const FFHpelRecord r = recs[ri];
    const int w = 16 >> r.sidx, no_rnd = r.tab >= 2;
    // avg_pixels2_xy2 stores without averaging in the reference ("FIXME non put", hpeldsp.c:151): keep the quirk
    const int avg = (r.tab & 1) && !(r.sidx == 3 && r.dxy == 3);
    for (int it = lane; it < w * r.h; it += 32) {
        const int x = it % w, y = it / w;
        const uint8_t *p = src + r.src_off + y * st + x;
        int v;
        switch (r.dxy) {
        case 0: v = p[0]; break;
        case 1: v = (p[0] + p[1] + 1 - no_rnd) >> 1; break;
        case 2: v = (p[0] + p[st] + 1 - no_rnd) >> 1; break;
        default: v = (p[0] + p[1] + p[st] + p[st + 1] + 2 - no_rnd) >> 2; break;
        }
        uint8_t *d = dst + r.dst_off + y * st + x;
        *d = (uint8_t)(avg ? (*d + v + 1) >> 1 : v);          // the fold into dst always rounds (op_avg = rnd_avg32, :330)
    }
}

// ---------------------------------------------------------------------------------------------------
// one thread per block, int16 write-back between the passes kept
template <int WHICH>
__global__ void __launch_bounds__(128) fdct_kernel(int16_t *__restrict__ blocks, size_t n)
{
    size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    int16_t *b = blocks + 64 * i;
    int m[8][8];
    fdct_load<WHICH>(b, m);
#pragma unroll
    for (int r = 0; r < 8; r++)
        reinterpret_cast<uint4 *>(b)[r] = make_uint4(pack16(m[r][0], m[r][1]), pack16(m[r][2], m[r][3]), pack16(m[r][4], m[r][5]), pack16(m[r][6], m[r][7]));
}

// PixblockDSPContext.get_pixels / diff_pixels (pixblockdsp_template.c:24-66), optionally followed by the forward DCT of
// fdct_kernel in the same thread: the 8x8 samples never exist as an int16 block in memory.  FDCT < 0: store them.
template <int FDCT>
__global__ void __launch_bounds__(128)
pixblock_kernel(const uint8_t *__restrict__ s1, const uint8_t *__restrict__ s2, const uint32_t *__restrict__ off1,
                const uint32_t *__restrict__ off2, ptrdiff_t stride, int16_t *__restrict__ blocks, size_t n)
{
    size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const uint8_t *a = s1 + off1[i], *b = s2 ? s2 + (off2 ? off2[i] : off1[i]) : nullptr;
    int m[8][8];
    pixblock_fetch<FDCT>(a, b, stride, m);
    int16_t *d = blocks + 64 * i;
#pragma unroll
    for (int r = 0; r < 8; r++)
        reinterpret_cast<uint4 *>(d)[r] = make_uint4(pack16(m[r][0], m[r][1]), pack16(m[r][2], m[r][3]), pack16(m[r][4], m[r][5]), pack16(m[r][6], m[r][7]));
}

// QpelDSPContext: MPEG-4 quarter-pel MC (libavcodec/qpeldsp.c:39-700), warp per record.  The (N+1) x (N+1) source patch
// goes to shared memory, then the horizontal phase plane Hx (N+1 rows, 8-bit after its own rounding, exactly the C code's
// halfH), then every lane finishes its pixels with the vertical phase: one formula for all 16 positions, 8-tap
// (-1 3 -6 20 20 -6 3 -1) with the sample index mirrored at both ends of the block.
struct QpelSmem { uint8_t f[17 * 20]; uint8_t hx[17 * 16]; };

template <int N>
__device__ __forceinline__ int qpel8tap(const uint8_t *s, int step, int i)
{
    auto m = [&](int j) { return (int)s[(j < 0 ? -1 - j : j > N ? 2 * N + 1 - j : j) * step]; };
    return (m(i) + m(i + 1)) * 20 - (m(i - 1) + m(i + 2)) * 6 + (m(i - 2) + m(i + 3)) * 3 - (m(i - 3) + m(i + 4));
}

template <int N>
__device__ __forceinline__ void qpel_record(QpelSmem &S, const FFQpelRecord &r, uint8_t *__restrict__ dst, const uint8_t *__restrict__ src,
                                            ptrdiff_t stride, int lane)
{
    const int x = r.mc & 3, y = r.mc >> 2, rnd = r.kind == 1 ? 15 : 16, up = r.kind == 1 ? 0 : 1;
    const int rows = y ? N + 1 : N, cols = x ? N + 1 : N;
    const uint8_t *sp = src + r.src_off;
    for (int i = lane; i < rows * cols; i += 32) { const int rr = i / cols, cc = i - rr * cols; S.f[rr * 20 + cc] = sp[rr * stride + cc]; }
    __syncwarp();
    for (int i = lane; i < rows * N; i += 32) {
        const int rr = i / N, cc = i % N;
        int v = S.f[rr * 20 + cc];
        if (x) {
            const int h = clip_u8((qpel8tap<N>(&S.f[rr * 20], 1, cc) + rnd) >> 5);
            v = x == 2 ? h : (S.f[rr * 20 + cc + (x == 3)] + h + up) >> 1;
        }
        S.hx[rr * 16 + cc] = (uint8_t)v;
    }
    __syncwarp();
    uint8_t *dp = dst + r.dst_off;
    for (int i = lane; i < N * N; i += 32) {
        const int rr = i / N, cc = i % N;
        int v = S.hx[rr * 16 + cc];
        if (y) {
            const int vv = clip_u8((qpel8tap<N>(&S.hx[cc], 16, rr) + rnd) >> 5);
            v = y == 2 ? vv : (S.hx[(rr + (y == 3)) * 16 + cc] + vv + up) >> 1;
        }
        uint8_t *d = dp + rr * stride + cc;
        *d = (uint8_t)(r.kind == 2 ? (*d + v + 1) >> 1 : v);
    }
}

__global__ void __launch_bounds__(128)
mpeg4_qpel_kernel(const FFQpelRecord *__restrict__ recs, size_t n, uint8_t *__restrict__ dst, const uint8_t *__restrict__ src, ptrdiff_t stride)
{
    __shared__ QpelSmem sm[4];
    const int lane = threadIdx.x & 31;
    const size_t ri = (size_t)blockIdx.x * 4 + (threadIdx.x >> 5);
    if (ri >= n) return;
    const FFQpelRecord r = recs[ri];
    if (r.sidx) qpel_record<8>(sm[threadIdx.x >> 5], r, dst, src, stride, lane);
    else        qpel_record<16>(sm[threadIdx.x >> 5], r, dst, src, stride, lane);
}

// Encoder-state metrics that only need the DSP tables (me_cmp.c:538-621): kind 11 dct_sad, 12 dct_max (diff_pixels ->
// FDCTDSPContext.fdct -> sum / max of |coefficient|; dxy selects the transform: 6 FAAN, 2 ifast, any other islow), 13 dct264_sad (diff ->
// H.264 8x8 forward transform rows then columns -> sum of |result|).  Warp per record, one lane per 8x8 quadrant.
__device__ __forceinline__ void dct264_1d(const int (&v)[8], int (&o)[8])
{
    const int s07 = v[0] + v[7], s16 = v[1] + v[6], s25 = v[2] + v[5], s34 = v[3] + v[4];
    const int a0 = s07 + s34, a1 = s16 + s25, a2 = s07 - s34, a3 = s16 - s25;
    const int d07 = v[0] - v[7], d16 = v[1] - v[6], d25 = v[2] - v[5], d34 = v[3] - v[4];
    const int a4 = d16 + d25 + (d07 + (d07 >> 1)), a5 = d07 - d34 - (d25 + (d25 >> 1));
    const int a6 = d07 + d34 - (d16 + (d16 >> 1)), a7 = d16 - d25 + (d34 + (d34 >> 1));
    o[0] = a0 + a1; o[1] = a4 + (a7 >> 2); o[2] = a2 + (a3 >> 1); o[3] = a5 + (a6 >> 2);
    o[4] = a0 - a1; o[5] = a6 - (a5 >> 2); o[6] = (a2 >> 1) - a3; o[7] = (a4 >> 2) - a7;
}

template <int T>   // T 0 islow, 2 ifast, 4 h264, 6 FAAN (ff_faandct)
__device__ __forceinline__ int dct_metric_block(const uint8_t *a, const uint8_t *b, ptrdiff_t st, bool want_max)
{
    int m[8][8];
    if constexpr (T == 6) {
        pixblock_fetch<6>(a, b, st, m);
        int s = 0;
#pragma unroll
        for (int k = 0; k < 64; k++) { const int v = (int)(int16_t)m[k >> 3][k & 7]; s = want_max ? max(s, iabs_m(v)) : s + iabs_m(v); }
        return s;
    }
#pragma unroll
    for (int r = 0; r < 8; r++) {
        int in[8], o[8];
#pragma unroll
        for (int k = 0; k < 8; k++) in[k] = a[r * st + k] - b[r * st + k];
        if (T == 0) islow_1d<4, 9>(in, o); else if (T == 2) ifast_1d(in, o); else dct264_1d(in, o);
#pragma unroll
        for (int k = 0; k < 8; k++) m[r][k] = (int)(int16_t)o[k];
    }
    int s = 0;
#pragma unroll
    for (int c = 0; c < 8; c++) {
        int in[8], o[8];
#pragma unroll
        for (int k = 0; k < 8; k++) in[k] = m[k][c];
        if (T == 0) islow_1d<-4, 17>(in, o); else if (T == 2) ifast_1d(in, o); else dct264_1d(in, o);
#pragma unroll
        for (int k = 0; k < 8; k++) { const int v = T == 4 ? o[k] : (int)(int16_t)o[k]; s = want_max ? max(s, iabs_m(v)) : s + iabs_m(v); }
    }
    return s;
}

__global__ void __launch_bounds__(128)
me_cmp_dct_kernel(int kind, int sidx, int fdct_sel, const uint8_t *__restrict__ cur, const uint8_t *__restrict__ ref, ptrdiff_t st, int h,
                  const FFMECmpRecord *__restrict__ recs, size_t n, int32_t *__restrict__ out)
{
    const int lane = threadIdx.x & 31;
    size_t ri = (size_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    if (ri >= n) return;
    const int nblk = sidx == 0 ? (h == 16 ? 4 : 2) : 1;
    int s = 0;
    if (lane < nblk) {
        const uint8_t *a = cur + recs[ri].cur_off + (lane & 1) * 8 + (lane >> 1) * 8 * st, *b = ref + recs[ri].ref_off + (lane & 1) * 8 + (lane >> 1) * 8 * st;
        if (kind == 13) s = dct_metric_block<4>(a, b, st, false);
        else if (fdct_sel == 2) s = dct_metric_block<2>(a, b, st, kind == 12);
        else if (fdct_sel == 6) s = dct_metric_block<6>(a, b, st, kind == 12);
        else s = dct_metric_block<0>(a, b, st, kind == 12);
    }
    s = warp_sum(s);
    if (lane == 0) out[ri] = s;
}

static int warps_grid(size_t n, int warps_per_cta) { return (int)((n + warps_per_cta - 1) / warps_per_cta); }

}  // namespace avb

using namespace avb;
extern "C" {

int ff_me_cmp_batch_cuda(int kind, int sidx, int dxy, const uint8_t *cur, const uint8_t *ref, ptrdiff_t stride, int h,
                         const FFMECmpRecord *recs, size_t n, int32_t *out, void *stream)
{
    avb::enter();
    if (!n) return 0;
    const bool ok = (kind == 0 && sidx <= 1 && dxy >= 0 && dxy <= 3) || (kind == 1 && sidx <= 1) || (kind == 2 && sidx <= 2) ||
                    ((kind == 3 || kind == 7) && sidx <= 1) || ((kind == 4 || kind == 5) && sidx == 0) || (kind == 6 && sidx <= 1) ||
                    ((kind == 8 || kind == 9) && sidx <= 1) || kind == 10 || (kind >= 11 && kind <= 13 && sidx <= 1 && (h == 8 || (h == 16 && sidx == 0)));
    if (!ok || sidx < 0) { set_error_msg("me_cmp_batch", "this (kind, size) slot is NULL in the reference table as well"); return -1; }
    if (kind >= 11) me_cmp_dct_kernel<<<warps_grid(n, 4), 128, 0, (cudaStream_t)stream>>>(kind, sidx, dxy, cur, ref, stride, h, recs, n, out);
    else me_cmp_kernel<<<warps_grid(n, 4), 128, 0, (cudaStream_t)stream>>>(kind, sidx, dxy, cur, ref, stride, h, recs, n, out);
    return check_launch("me_cmp_batch");
}

int ff_full_search_cuda(const uint8_t *cur, const uint8_t *ref, int stride, int w, int h, int range, int mb_y0, int mb_y1,
                        int32_t *out, void *stream)
{
    avb::enter();
    if (mb_y1 <= mb_y0) return 0;
    if (range != FS_R) { set_error_msg("full_search", "only me_range 16 is built"); return -1; }
    if ((w & 15) || (h & 15) || (stride & 15) || ((uintptr_t)cur & 15)) { set_error_msg("full_search", "picture must be MB aligned, cur 16-byte aligned"); return -1; }
    full_search_kernel_v2<<<dim3(w >> 4, mb_y1 - mb_y0), 256, 0, (cudaStream_t)stream>>>(cur, ref, stride, w, h, mb_y0, out);
    return check_launch("full_search");
}

int ff_hpel_batch_cuda(const FFHpelRecord *recs, size_t n, uint8_t *dst, const uint8_t *src, ptrdiff_t stride, void *stream)
{
    avb::enter();
    if (!n) return 0;
    hpel_kernel<<<warps_grid(n, 4), 128, 0, (cudaStream_t)stream>>>(recs, n, dst, src, stride);
    return check_launch("hpel_batch");
}

int ff_fdct_batch_cuda(int which, int16_t *blocks, size_t n, void *stream)
{
    avb::enter();
    using avb::fdct10_launch;
    if (!n) return 0;
    const int grid = (int)((n + 127) / 128);
    cudaStream_t st = (cudaStream_t)stream;
    switch (which) {
    case 0: fdct_kernel<0><<<grid, 128, 0, st>>>(blocks, n); break;
    case 1: fdct_kernel<1><<<grid, 128, 0, st>>>(blocks, n); break;
    case 2: fdct_kernel<2><<<grid, 128, 0, st>>>(blocks, n); break;
    case 3: fdct_kernel<3><<<grid, 128, 0, st>>>(blocks, n); break;
    case 4: case 5: return fdct10_launch(which, blocks, n, st);          // the 10-bit instances, fdct10.cu
    case 6: case 7: return avb::faan_fdct_launch(which, blocks, n, st);   // ff_faandct / ff_faandct248, faan_idct.cu
    default: set_error_msg("fdct_batch", "bad transform selector"); return -1;
    }
    return check_launch("fdct_batch");
}

int ff_mpeg4_qpel_batch_cuda(const FFQpelRecord *recs, size_t n, uint8_t *dst, const uint8_t *src, ptrdiff_t stride, void *stream)
{
    avb::enter();
    if (!n) return 0;
    mpeg4_qpel_kernel<<<warps_grid(n, 4), 128, 0, (cudaStream_t)stream>>>(recs, n, dst, src, stride);
    return check_launch("mpeg4_qpel_batch");
}

int ff_pixblock_fdct_batch_cuda(int which_fdct, const uint8_t *s1, const uint8_t *s2, const uint32_t *off1, const uint32_t *off2,
                                ptrdiff_t stride, int16_t *blocks, size_t n, void *stream)
{
    avb::enter();
    if (!n) return 0;
    if (!s1 || !off1 || !blocks || ((uintptr_t)blocks & 15)) { set_error_msg("pixblock_fdct_batch", "need s1, off1 and 16-byte aligned blocks"); return -1; }
    const int grid = (int)((n + 127) / 128);
    cudaStream_t st = (cudaStream_t)stream;
    switch (which_fdct) {
    case 0: pixblock_kernel<0><<<grid, 128, 0, st>>>(s1, s2, off1, off2, stride, blocks, n); break;
    case 1: pixblock_kernel<1><<<grid, 128, 0, st>>>(s1, s2, off1, off2, stride, blocks, n); break;
    case 2: pixblock_kernel<2><<<grid, 128, 0, st>>>(s1, s2, off1, off2, stride, blocks, n); break;
    case 3: pixblock_kernel<3><<<grid, 128, 0, st>>>(s1, s2, off1, off2, stride, blocks, n); break;
    case 6: pixblock_kernel<6><<<grid, 128, 0, st>>>(s1, s2, off1, off2, stride, blocks, n); break;
    case 7: pixblock_kernel<7><<<grid, 128, 0, st>>>(s1, s2, off1, off2, stride, blocks, n); break;
    default:
        if (which_fdct >= 0) { set_error_msg("pixblock_fdct_batch", "bad transform selector"); return -1; }
        pixblock_kernel<-1><<<grid, 128, 0, st>>>(s1, s2, off1, off2, stride, blocks, n); break;
    }
    return check_launch("pixblock_fdct_batch");
}

}  // extern "C"
