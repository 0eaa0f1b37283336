// libav_b200/csrc/prores.cu -- ProRes reconstruction: ProresDSPContext.idct_put (prores_idct_put_c, libavcodec/proresdsp.c:55-68) as a
// batched entry point and a table slot, and the decoder's whole-picture flush point (decode_slice_plane's idct_put calls of every slice of
// a picture, proresdec.c:425-482).
//
// One block: block[i] *= qmat[i] (int16 wrap), ff_prores_idct (simple_idct.c:222-234: the 10-bit row pass with extra_shift 2, whose
// DC-only test sees the dequantised values, then idctSparseCol_10 in place), then av_clip(block[i] + 512, 4, 1019) into 16-bit samples.
// The transform is the 10-bit IDCT's (idct10.cuh) with the ProresRows policy.  Both passes' results fit int16 (an int shifted right by 17 /
// 20), so the block the C function leaves is exactly the column pass's output.
//
// The batched and picture paths run a staged kernel on the WarpBlockStage layout of the 10-bit IDCT; unaligned blocks or pitches run a
// thread-per-block kernel whose threads never communicate, so the file also compiles for tests/hostsim/ (the picture addressing included).
#include "common.cuh"
#include "scratch.h"
#include "idct10.cuh"
#ifndef AVB_HOSTSIM
#include "block_stage.cuh"
#endif
#include "prores.cuh"
#include <string.h>

namespace avb {
namespace {

constexpr int PR_WARPS = 4;
constexpr int PR_PICS_PER_LAUNCH = 16;          // 16 x 224 bytes of kernel parameters

struct PrBatch {
    int16_t *blocks;
    uint8_t *frame;
    const uint32_t *dst_off;
    ptrdiff_t stride;
    const int16_t *qmats;
    const uint32_t *qidx;
    size_t n;
};
// the kernel's view of one picture (checked on the host)
struct PrPic {
    uint8_t *plane[3];
    ptrdiff_t ls[3];
    int mb_w, swf, c444, nxs, n_slices;
    const FFProresSlice *slices;
    const int16_t *blocks;
    size_t n_blocks;
    uint8_t qm[2][64];
};
// ST: the whole-packet decoder's launch (prores_dec.cu), which adds per picture its slices' plane status (prores.cuh)
template <bool ST> struct PrLaunch { PrPic pic[PR_PICS_PER_LAUNCH]; };
template <> struct PrLaunch<true> { PrPic pic[PR_PICS_PER_LAUNCH]; const uint32_t *status[PR_PICS_PER_LAUNCH]; };
__device__ __forceinline__ const uint32_t *pr_status(const PrLaunch<false> &, int) { return nullptr; }
__device__ __forceinline__ const uint32_t *pr_status(const PrLaunch<true> &L, int k) { return L.status[k]; }

// block i of a picture's coefficient buffer -> its destination and which matrix / scale factor dequantise it; false: no slice holds it, or
// (ST) its slice does not write its plane
template <bool ST>
__device__ __forceinline__ bool pr_locate(const PrPic &P, const uint32_t *status, size_t i, uint8_t *&dst, ptrdiff_t &ls, int &chroma, int &sf)
{
    // The decoder stages its slices back to back in slice order, so block i's slice follows from the geometry; one load confirms it.
    // Any other table takes a binary search for the last slice whose first block is <= i.
    const unsigned bpm = 4u + (P.c444 ? 8u : 4u), row_blocks = (unsigned)P.mb_w * bpm, full_blocks = bpm << P.swf;
    const unsigned ii = (unsigned)i, srow = ii / row_blocks;
    unsigned off = ii - srow * row_blocks, col = off / full_blocks;
    const unsigned nfull = (unsigned)(P.mb_w >> P.swf);
    if (col >= nfull) {
        col = nfull; off -= nfull * full_blocks;
        for (int b = 2; b >= 0; b--) {
            if (!((P.mb_w >> b) & 1) || b >= P.swf) continue;
            if (off < (bpm << b)) break;
            off -= bpm << b; col++;
        }
    } else off -= col * full_blocks;
    int lo = (int)(srow * (unsigned)P.nxs + col);
    if (lo >= P.n_slices || P.slices[lo].first_block != ii - off) {
        lo = 0;
        int hi = P.n_slices - 1;
        while (lo < hi) {
            const int mid = (lo + hi + 1) >> 1;
            if (P.slices[mid].first_block <= i) lo = mid; else hi = mid - 1;
        }
    }
    const FFProresSlice s = P.slices[lo];
    if (s.first_block > i) return false;
    const int sy = lo / P.nxs, sc = lo - sy * P.nxs, full = P.mb_w >> P.swf;
    int x, w;
    if (sc < full) { x = sc << P.swf; w = 1 << P.swf; }
    else {                                                           // the right edge: the set bits of the remainder, largest first
        x = full << P.swf; w = 0;
        int k = sc - full;
        for (int b = 2; b >= 0; b--) {
            if (!((P.mb_w >> b) & 1) || b >= P.swf) continue;
            if (k == 0) { w = 1 << b; break; }
            x += 1 << b; k--;
        }
    }
    const size_t jj = i - s.first_block;
    const int cshift = P.c444 ? 2 : 1, ny = 4 * w, nc = w << cshift;
    if (jj >= (size_t)(ny + 2 * nc)) return false;
    int j = (int)jj, p, mb, dx, dy, mbw;
    if (j < ny) { p = 0; mb = j >> 2; dx = (j & 1) * 8; dy = (j & 2) * 4; mbw = 16; }
    else {
        j -= ny; p = 1;
        if (j >= nc) { j -= nc; p = 2; }
        mb = j >> cshift;
        const int pos = j & ((1 << cshift) - 1);
        if (P.c444) { dx = (pos >> 1) * 8; dy = (pos & 1) * 8; mbw = 16; }   // TL, BL, TR, BR
        else        { dx = 0; dy = pos * 8; mbw = 8; }                       // top, bottom
    }
    if (ST && !pr_plane_written(status[lo], p)) return false;
    ls = P.ls[p];
    dst = P.plane[p] + (ptrdiff_t)(sy * 16 + dy) * ls + (ptrdiff_t)(((x + mb) * mbw + dx) * 2);
    chroma = p != 0;
    sf = s.sf;
    return true;
}

__device__ __forceinline__ uint32_t pr_mul2(uint32_t a, uint32_t q) { return pack16(lo16s(a) * lo16s(q), hi16s(a) * hi16s(q)); }
__device__ __forceinline__ uint4 pr_dequant(uint4 r, uint4 q) { return make_uint4(pr_mul2(r.x, q.x), pr_mul2(r.y, q.y), pr_mul2(r.z, q.z), pr_mul2(r.w, q.w)); }
// row r of (int16_t)(qm[k] * sf), packed like a coefficient row
__device__ __forceinline__ uint4 pr_qrow(const uint8_t *qm, int sf)
{
    uint32_t v[4];
#pragma unroll
    for (int k = 0; k < 4; k++) v[k] = pack16(qm[2 * k] * sf, qm[2 * k + 1] * sf);
    return make_uint4(v[0], v[1], v[2], v[3]);
}
__device__ __forceinline__ uint32_t pr_put2(uint32_t v)
{
    return (uint32_t)min(max(lo16s(v) + 512, 4), 1019) | (uint32_t)min(max(hi16s(v) + 512, 4), 1019) << 16;
}
// dequantised rows -> the column pass's packed int16 results, row by row
__device__ __forceinline__ void pr_transform(uint4 (&row)[8], uint32_t (&o)[8][4])
{
#pragma unroll
    for (int r = 0; r < 8; r++) row[r] = i10_row<ProresRows>(row[r]);
#pragma unroll
    for (int c = 0; c < 4; c++) {
        uint32_t w[8];
#pragma unroll
        for (int r = 0; r < 8; r++) w[r] = c == 0 ? row[r].x : c == 1 ? row[r].y : c == 2 ? row[r].z : row[r].w;
        int lo[8], hi[8];
        i10_col<0>(w, lo);
        i10_col<1>(w, hi);
#pragma unroll
        for (int y = 0; y < 8; y++) o[y][c] = pack16(lo[y], hi[y]);
    }
}
__device__ __forceinline__ uint4 pr_load_row(const int16_t *g, int r)
{
    const int16_t *s = g + 8 * r;
    return make_uint4(pack16(s[0], s[1]), pack16(s[2], s[3]), pack16(s[4], s[5]), pack16(s[6], s[7]));
}
__device__ __forceinline__ void pr_store_samples(uint8_t *dst, ptrdiff_t ls, const uint32_t (&o)[8][4])
{
    for (int y = 0; y < 8; y++) {
        uint16_t *q = reinterpret_cast<uint16_t *>(dst + y * ls);
        for (int c = 0; c < 4; c++) { const uint32_t p = pr_put2(o[y][c]); q[2 * c] = (uint16_t)p; q[2 * c + 1] = (uint16_t)(p >> 16); }
    }
}

// ---- thread per block, 2-byte accesses: any alignment; the only kernels of the host build --------------------------------------------
__global__ void __launch_bounds__(128) prores_idct_block_kernel(const PrBatch B)
{
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= B.n) return;
    int16_t *g = B.blocks + 64 * i;
    const int16_t *q = B.qmats + 64 * (size_t)(B.qidx ? B.qidx[i] : 0);
    uint4 row[8];
    for (int r = 0; r < 8; r++) row[r] = pr_dequant(pr_load_row(g, r), pr_load_row(q, r));
    uint32_t o[8][4];
    pr_transform(row, o);
    for (int y = 0; y < 8; y++)
        for (int c = 0; c < 4; c++) { g[8 * y + 2 * c] = (int16_t)o[y][c]; g[8 * y + 2 * c + 1] = (int16_t)(o[y][c] >> 16); }
    pr_store_samples(B.frame + B.dst_off[i], B.stride, o);
}

template <bool ST>
__global__ void __launch_bounds__(128) prores_picture_block_kernel(const __grid_constant__ PrLaunch<ST> L)
{
    const PrPic &P = L.pic[blockIdx.y];
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= P.n_blocks) return;
    uint8_t *dst; ptrdiff_t ls; int chroma, sf;
    if (!pr_locate<ST>(P, pr_status(L, blockIdx.y), i, dst, ls, chroma, sf)) return;
    const int16_t *g = P.blocks + 64 * i;
    uint4 row[8];
    for (int r = 0; r < 8; r++) row[r] = pr_dequant(pr_load_row(g, r), pr_qrow(P.qm[chroma] + 8 * r, sf));
    uint32_t o[8][4];
    pr_transform(row, o);
    pr_store_samples(dst, ls, o);
}

#ifndef AVB_HOSTSIM
// ---- the staged kernels: simple_idct10_staged_kernel's layout (idct10.cu) ------------------------------------------------------------
// A warp owns 32 consecutive blocks: eight coalesced 512-byte cp.async requests into the XOR-swizzled tile (double-buffered), every lane
// transforms ITS block in registers.  Batch (PIC false): the result goes back through the tile as eight coalesced 512-byte stores, the
// samples leave as eight 16-byte rows per lane: 384 B per block.  Picture (PIC true, one picture per blockIdx.y): each lane derives its
// block's destination and matrix, before it waits for the group's coefficients so that the slice search overlaps their arrival; nothing
// goes back to the coefficients: 256 B per block.
template <bool PIC, bool ST = false>
__device__ __forceinline__ void pr_staged(const PrBatch *B, const PrPic *P, uint4 (&tile)[PR_WARPS][2][256], const uint8_t (*qm)[64],
                                          const uint32_t *status = nullptr)
{
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    int16_t *blocks = PIC ? const_cast<int16_t *>(P->blocks) : B->blocks;
    const size_t n = PIC ? P->n_blocks : B->n;
    const WarpBlockStage S(&tile[warp][0][0], lane);
    const size_t groups = (n + 31) / 32, gstride = (size_t)gridDim.x * PR_WARPS;
    size_t g = (size_t)blockIdx.x * PR_WARPS + warp;
    unsigned buf = 0;
    if (g < groups) S.issue(blocks, g, n, S.buffer(0));
    for (; g < groups; g += gstride, buf ^= 4096u) {
        const size_t gn = g + gstride;
        const unsigned tb = S.buffer(buf);
        if (gn < groups) S.issue(blocks, gn, n, S.buffer(buf ^ 4096u));
        const size_t i = g * 32 + lane;
        bool live = i < n;
        uint8_t *dst = nullptr;
        ptrdiff_t ls = PIC ? 0 : B->stride;
        int chroma = 0, sf = 0;
        const uint4 *q = nullptr;
        if (PIC) live = live && pr_locate<ST>(*P, status, i, dst, ls, chroma, sf);
        else {
            q = reinterpret_cast<const uint4 *>(B->qmats + 64 * (size_t)(live && B->qidx ? B->qidx[i] : 0));
            if (live) dst = B->frame + B->dst_off[i];
        }
        if (gn < groups) cp_async_wait<1>(); else cp_async_wait<0>();
        __syncwarp();
        uint4 row[8];
#pragma unroll
        for (int r = 0; r < 8; r++) row[r] = pr_dequant(S.row(tb, r), PIC ? pr_qrow(&qm[chroma][8 * r], sf) : __ldg(q + r));
        uint32_t o[8][4];
        pr_transform(row, o);
        if (!PIC) {
#pragma unroll
            for (int y = 0; y < 8; y++) S.put_row(tb, y, make_uint4(o[y][0], o[y][1], o[y][2], o[y][3]));
            S.flush(blocks, g, n, tb);
        }
        if (live) {
            if (!(((uintptr_t)dst | (uintptr_t)ls) & 15)) {
#pragma unroll
                for (int y = 0; y < 8; y++)
                    *reinterpret_cast<uint4 *>(dst + y * ls) = make_uint4(pr_put2(o[y][0]), pr_put2(o[y][1]), pr_put2(o[y][2]), pr_put2(o[y][3]));
            } else pr_store_samples(dst, ls, o);
        }
        __syncwarp();     // every lane is done with this buffer before the next group is requested into it
    }
}

__global__ void __launch_bounds__(PR_WARPS * 32) prores_idct_staged_kernel(const PrBatch B)
{
    __shared__ __align__(128) uint4 tile[PR_WARPS][2][256];
    pr_staged<false>(&B, nullptr, tile, nullptr);
}

template <bool ST>
__global__ void __launch_bounds__(PR_WARPS * 32) prores_picture_staged_kernel(const __grid_constant__ PrLaunch<ST> L)
{
    __shared__ __align__(128) uint4 tile[PR_WARPS][2][256];
    __shared__ __align__(16) uint8_t qm[2][64];
    const PrPic &P = L.pic[blockIdx.y];
    qm[threadIdx.x >> 6][threadIdx.x & 63] = P.qm[threadIdx.x >> 6][threadIdx.x & 63];
    __syncthreads();
    pr_staged<true, ST>(nullptr, &P, tile, qm, pr_status(L, blockIdx.y));
}

// resident CTAs of a staged kernel over the whole device: the persistent grids never exceed one wave
template <class K> unsigned pr_wave(K kernel)
{
    int per_sm = 0;
    if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kernel, PR_WARPS * 32, 0) != cudaSuccess || per_sm < 1) per_sm = 1;
    return (unsigned)(per_sm * sm_count());
}
#endif

int launch_prores_batch(const PrBatch &B, cudaStream_t st)
{
    if (!B.n) return 0;
#ifndef AVB_HOSTSIM
    if (!(((uintptr_t)B.blocks | (uintptr_t)B.qmats | (uintptr_t)B.stride) & 15)) {
        static const unsigned wave = pr_wave(prores_idct_staged_kernel);
        const size_t groups = (B.n + 31) / 32;
        const unsigned grid = (unsigned)min((size_t)wave, (groups + PR_WARPS - 1) / PR_WARPS);
        prores_idct_staged_kernel<<<grid, PR_WARPS * 32, 0, st>>>(B);
        return check_launch("ff_prores_idct_put_batch_cuda");
    }
#endif
    AVB_LAUNCH(prores_idct_block_kernel, dim3((unsigned)((B.n + 127) / 128)), dim3(128), 0, st)(B);
    return check_launch("ff_prores_idct_put_batch_cuda");
}

void pr_set_status(PrLaunch<false> &, int, const uint32_t *const *, int) {}
void pr_set_status(PrLaunch<true> &L, int k, const uint32_t *const *status, int i) { L.status[k] = status[i]; }

int pr_refuse(const char *msg) { set_error_msg("ff_prores_decode_pictures_cuda", msg); return -1; }

int pr_picture(const FFProresPictureWork &w, PrPic &P)
{
    if (w.chroma_format != 2 && w.chroma_format != 3) return pr_refuse("chroma_format must be 2 (4:2:2) or 3 (4:4:4)");
    if (w.slice_width_factor < 0 || w.slice_width_factor > 3) return pr_refuse("slice_width_factor must be 0..3");
    if (w.mb_width < 1 || w.mb_height < 1 || w.mb_width > 8192 || w.mb_height > 8192) return pr_refuse("macroblock dimensions outside 1..8192");
    const int c444 = w.chroma_format == 3;
    for (int p = 0; p < 3; p++) {
        if (!w.data[p] || ((uintptr_t)w.data[p] & 1)) return pr_refuse("NULL or odd plane pointer");
        if (w.linesize[p] <= 0 || (w.linesize[p] & 1)) return pr_refuse("linesize must be even and positive");
        const long need = (long)w.mb_width * (p == 0 || c444 ? 32 : 16);
        if (w.linesize[p] < need || w.mb_rows[p] < w.mb_height) return pr_refuse("plane too small for whole macroblocks");
    }
    const int nxs = pr_slices_per_row(w.mb_width, w.slice_width_factor);
    if ((long)w.n_slices != (long)nxs * w.mb_height) return pr_refuse("the slice table does not cover the picture");
    if (!w.slices || (w.n_blocks && !w.blocks)) return pr_refuse("NULL slice table or coefficient buffer");
    if (w.n_blocks > 0xffffffffu) return pr_refuse("more than 2^32 - 1 blocks");
    memset(&P, 0, sizeof(P));
    for (int p = 0; p < 3; p++) { P.plane[p] = w.data[p]; P.ls[p] = w.linesize[p]; }
    P.mb_w = w.mb_width; P.swf = w.slice_width_factor; P.c444 = c444; P.nxs = nxs; P.n_slices = w.n_slices;
    P.slices = w.slices; P.blocks = w.blocks; P.n_blocks = w.n_blocks;
    memcpy(P.qm[0], w.qmat_luma, 64); memcpy(P.qm[1], w.qmat_chroma, 64);
    return 0;
}

// pictures already checked by pr_picture; up to PR_PICS_PER_LAUNCH per launch, each picture one row (blockIdx.y) of the grid
template <bool ST>
int launch_pictures(const FFProresPictureWork *pictures, const uint32_t *const *status, int n, cudaStream_t st)
{
    for (int g0 = 0; g0 < n; g0 += PR_PICS_PER_LAUNCH) {
        const int m = n - g0 < PR_PICS_PER_LAUNCH ? n - g0 : PR_PICS_PER_LAUNCH;
        PrLaunch<ST> L;
        memset(&L, 0, sizeof(L));
        size_t most = 0;
        bool aligned = true;
        for (int k = 0; k < m; k++) {
            pr_picture(pictures[g0 + k], L.pic[k]);
            most = L.pic[k].n_blocks > most ? L.pic[k].n_blocks : most;
            aligned = aligned && !((uintptr_t)L.pic[k].blocks & 15);
            pr_set_status(L, k, status, g0 + k);
        }
        if (!most) continue;
#ifndef AVB_HOSTSIM
        if (aligned) {
            static const unsigned wave = pr_wave(prores_picture_staged_kernel<ST>);
            const size_t groups = (most + 31) / 32;
            const unsigned grid = (unsigned)max((size_t)1, min((size_t)(wave / (unsigned)m), (groups + PR_WARPS - 1) / PR_WARPS));
            prores_picture_staged_kernel<ST><<<dim3(grid, m), PR_WARPS * 32, 0, st>>>(L);
            if (check_launch("ff_prores_decode_pictures_cuda")) return -1;
            continue;
        }
#endif
        AVB_LAUNCH(prores_picture_block_kernel<ST>, dim3((unsigned)((most + 127) / 128), m), dim3(128), 0, st)(L);
        if (check_launch("ff_prores_decode_pictures_cuda")) return -1;
    }
    return 0;
}

// ProresDSPContext.idct_put: a batch of one with host pointers.  Device layout: [0,128) the block, [128,256) qmat, [256,260) the offset,
// [512, 512 + 8 * 16) the 8 x 8 samples at pitch 16 bytes.
void slot_prores_idct_put(uint16_t *out, ptrdiff_t linesize, int16_t *block, const int16_t *qmat)
{
    ScratchLock lk;
    Scratch &S = scratch();
    uint8_t *h = (uint8_t *)S.pinned2(4096), *d = (uint8_t *)S.dev(8, 4096);
    cudaStream_t *st = S.streams();
    if (!h || !d || !st) return;
    memcpy(h, block, 128);
    memcpy(h + 128, qmat, 128);
    const uint32_t off = 512;
    memcpy(h + 256, &off, 4);
    if (cudaMemcpyAsync(d, h, 260, cudaMemcpyHostToDevice, st[0]) != cudaSuccess) { set_error("prores slot:h2d", cudaGetLastError()); return; }
    PrBatch B = { (int16_t *)d, d, (const uint32_t *)(d + 256), 16, (const int16_t *)(d + 128), nullptr, 1 };
    if (launch_prores_batch(B, st[0])) return;
    if (cudaMemcpyAsync(h, d, 640, cudaMemcpyDeviceToHost, st[0]) != cudaSuccess || cudaStreamSynchronize(st[0]) != cudaSuccess) {
        set_error("prores slot:d2h", cudaGetLastError()); return;
    }
    memcpy(block, h, 128);
    uint8_t *dst = (uint8_t *)out;
    for (int y = 0; y < 8; y++) memcpy(dst + y * (linesize >> 1) * 2, h + 512 + 16 * y, 16);
}

}  // namespace

int launch_prores_pictures(const FFProresPictureWork *pictures, int n, cudaStream_t st, const uint32_t *const *status)
{
    return status ? launch_pictures<true>(pictures, status, n, st) : launch_pictures<false>(pictures, nullptr, n, st);
}

}  // namespace avb

using namespace avb;

extern "C" {

int ff_prores_idct_put_batch_cuda(int16_t *blocks, uint8_t *frame, const uint32_t *dst_off, ptrdiff_t stride, const int16_t *qmats,
                                  const uint32_t *qmat_idx, size_t n, void *stream)
{
    avb::enter();
    if ((n && (!blocks || !frame || !dst_off || !qmats)) || (stride & 1)) {
        set_error_msg("ff_prores_idct_put_batch_cuda", "bad argument"); return -1;
    }
    const PrBatch B = { blocks, frame, dst_off, stride, qmats, qmat_idx, n };
    return launch_prores_batch(B, (cudaStream_t)stream);
}

int ff_prores_decode_pictures_cuda(const FFProresPictureWork *pictures, int n, void *stream)
{
    avb::enter();
    if (n == 0) return 0;
    if (!pictures || n < 0) return pr_refuse("NULL pictures or a negative count");
    for (int k = 0; k < n; k++) {                  // every picture is checked before anything is launched
        PrPic P;
        if (pr_picture(pictures[k], P)) return -1;
    }
    return launch_prores_pictures(pictures, n, (cudaStream_t)stream);
}

void ff_proresdsp_init_cuda(ProresDSPContext *dsp)
{
    avb::enter();
    if (!dsp) return;
    dsp->idct_put = slot_prores_idct_put;
    dsp->idct_permutation_type = FF_IDCT_PERM_NONE;
    for (int i = 0; i < 64; i++) dsp->idct_permutation[i] = (uint8_t)i;     // ff_init_scantable_permutation() for FF_IDCT_PERM_NONE
}

}  // extern "C"
