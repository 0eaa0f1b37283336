// libav_b200/csrc/h264intra.cu -- batched H.264 intra reconstruction (SURVEY 8f rank 2): what hl_decode_mb() does for
// the intra macroblocks of a picture (libavcodec/h264_mb_template.c:40-, hl_decode_mb_predict_luma h264_mb.c:607-731,
// chroma :hl_decode_mb 158-197): intra prediction (H264PredContext) interleaved with the residual
// (h264_idct_add / dc_add / idct8 / add16intra / add8) block by block, because every block predicts from pixels the
// previous blocks just reconstructed.
//
// Dependencies reach left, up-left, up and up-right, so macroblock rows run as a wavefront: one warp per macroblock row,
// staying two macroblocks behind the row above (the same progress-flag scheme as the deblocking kernel).  A macroblock is
// reconstructed inside a shared-memory tile that also holds its neighbour row / column; prediction of a block runs one
// sample per lane from the edge arrays (h264pred.cuh), the residual reuses the device transforms of h264dsp.cuh.
// Non-intra macroblocks are left as the earlier passes (motion compensation + residual) wrote them; they only feed
// neighbour samples to the intra ones.
#include "h264pred.cuh"
#include "h264dsp.cuh"
#include "../../include/avdsp_b200.h"

namespace avb {

constexpr int LP = 32;        // luma tile: 17 rows x 32; sample (x, y) of the macroblock at [1 + y][4 + x]
constexpr int CP = 16;        // chroma tile: 9 rows x 16; sample (x, y) at [1 + y][4 + x]

__device__ __forceinline__ uint8_t ld_cg8(const uint8_t *p) { return __ldcg(p); }
__device__ __forceinline__ int s16i(int v) { return (int)(int16_t)v; }

// raw edges of the n x n block whose top-left sample is tile[r0][c0] (pitch P), gathered by the whole warp;
// `tr_ok`: the n samples to the top right exist (otherwise the last top sample is repeated, h264_mb.c:676-686)
template <int P>
__device__ __forceinline__ void gather_raw(IntraRaw &r, const uint8_t *tile, int r0, int c0, int n, bool tr_ok, int lane)
{
    const uint8_t *top = tile + (r0 - 1) * P + c0;
    if (lane < 16) { if (lane < n || n <= 8) r.top[lane] = top[(lane < n || tr_ok) ? lane : n - 1]; }
    else if (lane - 16 < n) r.left[lane - 16] = tile[(r0 + lane - 16) * P + c0 - 1];
    if (lane == 0) r.corner = top[-1];
}

// filtered 8x8 edges, one entry per lane (PREDICT_8x8_LOAD_*, h264pred_template.c:840-875)
__device__ __forceinline__ void edges8_parallel(IntraEdges &e, const IntraRaw &r, bool has_tl, bool has_tr, int lane)
{
    const uint8_t *t = r.top, *l = r.left;
    const int c = r.corner;
    if (lane < 16) {
        int v;
        if (lane == 0) v = ip_f3(has_tl ? c : t[0], t[0], t[1]);
        else if (lane < 7) v = ip_f3(t[lane - 1], t[lane], t[lane + 1]);
        else if (lane == 7) v = ip_f3(has_tr ? t[8] : t[7], t[7], t[6]);
        else if (!has_tr) v = t[7];
        else if (lane < 15) v = ip_f3(t[lane - 1], t[lane], t[lane + 1]);
        else v = (t[14] + 3 * t[15] + 2) >> 2;
        e.t[lane + 1] = v;
    } else if (lane < 24) {
        const int k = lane - 16;
        e.l[k + 1] = k == 0 ? ip_f3(has_tl ? c : l[0], l[0], l[1]) : k < 7 ? ip_f3(l[k - 1], l[k], l[k + 1]) : (l[6] + 3 * l[7] + 2) >> 2;
    } else if (lane == 24) {
        e.t[0] = e.l[0] = ip_f3(l[0], c, t[0]);
    }
}

// 4x4 residual on 16 lanes: lane (x = lane & 3, y = lane >> 2) owns pixel (x, y); returns the value to add (already >> 6)
__device__ __forceinline__ int idct4_lane(int16_t *co, int *tmp, int lane)
{
    const int i = lane & 3, k = lane >> 2;
    const int c0 = i == 0 ? s16i(co[0] + 32) : co[i], c1 = co[i + 4], c2 = co[i + 8], c3 = co[i + 12];
    const int z0 = c0 + c2, z1 = c0 - c2, z2 = (c1 >> 1) - c3, z3 = c1 + (c3 >> 1);
    tmp[i + 4 * k] = s16i(k == 0 ? z0 + z3 : k == 1 ? z1 + z2 : k == 2 ? z1 - z2 : z0 - z3);
    __syncwarp(0xffff);
    const int d0 = tmp[4 * i], d1 = tmp[4 * i + 1], d2 = tmp[4 * i + 2], d3 = tmp[4 * i + 3];
    const int y0 = d0 + d2, y1 = d0 - d2, y2 = (d1 >> 1) - d3, y3 = d1 + (d3 >> 1);
    co[lane] = 0;
    return (k == 0 ? y0 + y3 : k == 1 ? y1 + y2 : k == 2 ? y1 - y2 : y0 - y3) >> 6;
}

__global__ void __launch_bounds__(32)
h264_intra_kernel(const FFH264IntraMB *__restrict__ mbs, int mb_w, int rows_pp, int16_t *__restrict__ coeffs, size_t coeff_stride,
                  const uint8_t *__restrict__ nnzc_all, uint8_t *luma, uint8_t *cb, uint8_t *cr, int ls, int uvls, uint32_t *progress, uint32_t *ticket)
{
    __shared__ __align__(16) uint8_t Y[17 * LP];
    __shared__ __align__(16) uint8_t C[2][9 * CP];
    __shared__ __align__(16) int16_t co[2][768];          // this macroblock's coefficients / the next one's (prefetch)
    __shared__ __align__(16) FFH264IntraMB Ms[2];
    __shared__ __align__(16) uint8_t nz[2][128];
    __shared__ IntraRaw raw;
    __shared__ IntraEdges edges;
    __shared__ IntraBig big;
    __shared__ int tmp[64];
    // rows are handed out by an atomic ticket in the order CTAs START: whoever holds row r knows that row r - 1 has been taken by a CTA that
    // is running or done, whatever order the hardware dispatches block indices in
    const int lane = threadIdx.x;
    int row = 0;
    if (lane == 0) row = (int)atomicAdd(ticket, 1u);
    row = __shfl_sync(0xffffffffu, row, 0);
    const int prow = row % rows_pp;                                            // prow: row inside its picture
    volatile uint32_t *prog = progress;
    uint8_t *const cplane[2] = { cb, cr };
    const bool co16 = !(coeff_stride & 7) && !((uintptr_t)coeffs & 15);

    // side information and coefficients do not depend on other rows: fetch macroblock x + 1 while x is reconstructed
    auto fetch = [&](int x, int b) {
        const size_t m = (size_t)row * mb_w + x;
        if (lane < 6) cp_async4(reinterpret_cast<uint32_t *>(&Ms[b]) + lane, reinterpret_cast<const uint32_t *>(&mbs[m]) + lane);
        if (lane < 30) cp_async4(reinterpret_cast<uint32_t *>(nz[b]) + lane, reinterpret_cast<const uint32_t *>(nnzc_all + m * 120) + lane);
        const int16_t *src = coeffs + m * coeff_stride;
        if (co16) { for (int i = lane; i < 96; i += 32) cp_async16(reinterpret_cast<uint4 *>(co[b]) + i, reinterpret_cast<const uint4 *>(src) + i, true); }
        else      { for (int i = lane; i < 384; i += 32) cp_async4(reinterpret_cast<uint32_t *>(co[b]) + i, reinterpret_cast<const uint32_t *>(src) + i); }
        cp_async_commit();
    };
    fetch(0, 0);

    for (int x = 0; x < mb_w; x++) {
        const int cur = x & 1;
        if (x + 1 < mb_w) { fetch(x + 1, cur ^ 1); cp_async_wait<1>(); } else cp_async_wait<0>();
        __syncwarp();
        const FFH264IntraMB &M = Ms[cur];
        const uint8_t *nnzc = nz[cur];
        int16_t *mb = co[cur];
        const size_t m = (size_t)row * mb_w + x;
        // only an intra macroblock reads the row above; the others neither wait for it nor look at it
        const bool needs_above = prow > 0 && M.kind != 0;
        if (needs_above) {
            if (lane == 0) { const uint32_t need = min(x + 2, mb_w); while (prog[row - 1] < need) { } }
            __syncwarp();
        }
        // the previous macroblock's last column becomes this one's left column (tile column 3)
        if (x > 0) {
            if (lane < 17) Y[lane * LP + 3] = Y[lane * LP + 19];
            if (lane < 18) { const int p = lane / 9, r = lane % 9; C[p][r * CP + 3] = C[p][r * CP + 11]; }
        }
        __syncwarp();
        // row above: samples x = -1 .. 23 (the corner, this macroblock's 16, and 8 of the macroblock up-right)
        if (needs_above) {
            const uint8_t *g = luma + (size_t)(row * 16 - 1) * ls + x * 16;
            if (lane < 6 && (lane < 4 || x + 1 < mb_w)) *reinterpret_cast<uint32_t *>(&Y[4 + 4 * lane]) = __ldcg(reinterpret_cast<const uint32_t *>(g) + lane);
            if (lane >= 8 && lane < 12) {
                const int p = (lane >> 1) & 1, q = lane & 1;
                *reinterpret_cast<uint32_t *>(&C[p][4 + 4 * q]) = __ldcg(reinterpret_cast<const uint32_t *>(cplane[p] + (size_t)(row * 8 - 1) * uvls + x * 8) + q);
            }
            if (lane == 31) Y[3] = x > 0 ? ld_cg8(g - 1) : 0;
            if (lane == 30) C[0][3] = x > 0 ? ld_cg8(cb + (size_t)(row * 8 - 1) * uvls + x * 8 - 1) : 0;
            if (lane == 29) C[1][3] = x > 0 ? ld_cg8(cr + (size_t)(row * 8 - 1) * uvls + x * 8 - 1) : 0;
        }
        const int kind = M.kind;
        if (kind == 0) {
            // not ours: only its last column is needed (by the macroblock to the right); the row below re-reads from memory
            for (int i = lane; i < 64; i += 32)
                *reinterpret_cast<uint32_t *>(&Y[(1 + (i >> 2)) * LP + 4 + 4 * (i & 3)]) = __ldcg(reinterpret_cast<const uint32_t *>(luma + (size_t)(row * 16 + (i >> 2)) * ls + x * 16) + (i & 3));
            {
                const int p = lane >> 4, r = (lane >> 1) & 7, q = lane & 1;
                *reinterpret_cast<uint32_t *>(&C[p][(1 + r) * CP + 4 + 4 * q]) = __ldcg(reinterpret_cast<const uint32_t *>(cplane[p] + (size_t)(row * 8 + r) * uvls + x * 8) + q);
            }
            __syncwarp();
        } else {
            __syncwarp();
            if (kind == 1) {                                   // intra 4x4: 16 blocks in coding order
                for (int i = 0; i < 16; i++) {
                    const int bx = (i & 1) + 2 * ((i >> 2) & 1), by = ((i >> 1) & 1) + 2 * (i >> 3);
                    const int mode = M.mode4[i], r0 = 1 + 4 * by, c0 = 4 + 4 * bx;
                    const bool tr_ok = (M.topright_samples_available << i) & 0x8000;
                    // edge arrays straight from the tile: lanes 0..8 -> T(-1..7), lanes 16..20 -> L(-1..3)
                    if (lane < 9) edges.t[lane] = Y[(r0 - 1) * LP + c0 - 1 + ((lane < 5 || tr_ok) ? lane : 4)];
                    else if (lane >= 16 && lane < 21) edges.l[lane - 16] = Y[(r0 - 1 + lane - 16) * LP + c0 - 1];
                    __syncwarp();
                    const int nnz = nnzc[scan8_of(i)];
                    int16_t *blk = mb + 16 * i;
                    const bool dc_only = nnz == 1 && blk[0];
                    if (lane < 16) {
                        int v = intra_directional(edges, 4, mode, lane & 3, lane >> 2);
                        if (nnz) {
                            if (dc_only) v = clip_u8(v + ((blk[0] + 32) >> 6));
                            else v = clip_u8(v + idct4_lane(blk, tmp, lane));
                        }
                        Y[(r0 + (lane >> 2)) * LP + c0 + (lane & 3)] = (uint8_t)v;
                    }
                    __syncwarp();
                    if (dc_only && lane == 0) blk[0] = 0;
                }
            } else if (kind == 2) {                            // intra 8x8
                for (int k = 0; k < 4; k++) {
                    const int i = 4 * k, bx = k & 1, by = k >> 1, mode = M.mode4[i];
                    const bool tl = (M.topleft_samples_available << i) & 0x8000, tr = (M.topright_samples_available << i) & 0x4000;
                    gather_raw<LP>(raw, Y, 1 + 8 * by, 4 + 8 * bx, 8, tr, lane);
                    __syncwarp();
                    edges8_parallel(edges, raw, tl, tr, lane);
                    __syncwarp();
                    for (int s = lane; s < 64; s += 32)
                        Y[(1 + 8 * by + (s >> 3)) * LP + 4 + 8 * bx + (s & 7)] = (uint8_t)intra_directional(edges, 8, mode, s & 7, s >> 3);
                    __syncwarp();
                    const int nnz = nnzc[scan8_of(i)];
                    int16_t *blk = mb + 16 * i;
                    uint8_t *d = &Y[(1 + 8 * by) * LP + 4 + 8 * bx];
                    if (nnz) {
                        if (nnz == 1 && blk[0]) {
                            const int dc = (blk[0] + 32) >> 6;
                            for (int s = lane; s < 64; s += 32) { uint8_t *q = d + (s >> 3) * LP + (s & 7); *q = (uint8_t)clip_u8(*q + dc); }
                            __syncwarp();
                            if (lane == 0) blk[0] = 0;
                        } else {
                            // column pass on 8 lanes, row pass on 8 lanes (h264idct_template.c:69-141), int16 round trip kept
                            if (lane == 0) blk[0] = (int16_t)(blk[0] + 32);
                            __syncwarp();
                            if (lane < 8) {
                                int v[8], o[8];
#pragma unroll
                                for (int q = 0; q < 8; q++) v[q] = blk[lane + 8 * q];
                                h264_idct8_1d(v, o);
#pragma unroll
                                for (int q = 0; q < 8; q++) blk[lane + 8 * q] = (int16_t)o[q];
                            }
                            __syncwarp();
                            if (lane < 8) {
                                int v[8], o[8];
#pragma unroll
                                for (int q = 0; q < 8; q++) v[q] = blk[8 * lane + q];
                                h264_idct8_1d(v, o);
#pragma unroll
                                for (int q = 0; q < 8; q++) d[lane + q * LP] = (uint8_t)clip_u8(d[lane + q * LP] + (o[q] >> 6));
                            }
                            __syncwarp();
                            blk[lane] = 0; blk[lane + 32] = 0;
                        }
                    }
                    __syncwarp();
                }
            } else {                                           // intra 16x16, then h264_idct_add16intra
                gather_raw<LP>(raw, Y, 1, 4, 16, false, lane);
                __syncwarp();
                if (lane == 0) intra_big_prepare(big, raw, 16);
                __syncwarp();
                for (int s = lane; s < 256; s += 32) Y[(1 + (s >> 4)) * LP + 4 + (s & 15)] = (uint8_t)intra_big_sample(big, raw, 16, M.mode16, s & 15, s >> 4);
                __syncwarp();
                if (lane < 16) {
                    const int bx = (lane & 1) + 2 * ((lane >> 2) & 1), by = ((lane >> 1) & 1) + 2 * (lane >> 3);
                    uint8_t *d = &Y[(1 + 4 * by) * LP + 4 + 4 * bx];
                    if (nnzc[scan8_of(lane)]) h264_idct4_add(d, mb + 16 * lane, LP); else if (mb[16 * lane]) h264_dc_add(d, mb + 16 * lane, LP, 4);
                }
                __syncwarp();
            }
            // chroma: pred8x8 on both planes, then h264_idct_add8
            for (int p = 0; p < 2; p++) {
                gather_raw<CP>(raw, C[p], 1, 4, 8, false, lane);
                __syncwarp();
                if (lane == 0) intra_big_prepare(big, raw, 8);
                __syncwarp();
                for (int s = lane; s < 64; s += 32) C[p][(1 + (s >> 3)) * CP + 4 + (s & 7)] = (uint8_t)intra_big_sample(big, raw, 8, M.chroma_mode, s & 7, s >> 3);
                __syncwarp();
            }
            if (M.chroma_residual && lane < 8) {
                const int p = lane >> 2, k = lane & 3, i = 16 + 16 * p + k;
                uint8_t *d = &C[p][(1 + 4 * (k >> 1)) * CP + 4 + 4 * (k & 1)];
                if (nnzc[scan8_of(i)]) h264_idct4_add(d, mb + 16 * i, CP); else if (mb[16 * i]) h264_dc_add(d, mb + 16 * i, CP, 4);
            }
            __syncwarp();
            // write the macroblock and its (now partly zeroed) coefficients back
            for (int i = lane; i < 64; i += 32) {
                const int r = i >> 2, q = i & 3;
                *reinterpret_cast<uint32_t *>(luma + (size_t)(row * 16 + r) * ls + x * 16 + 4 * q) = *reinterpret_cast<const uint32_t *>(&Y[(1 + r) * LP + 4 + 4 * q]);
            }
            {
                const int p = lane >> 4, r = (lane >> 1) & 7, q = lane & 1;
                *reinterpret_cast<uint32_t *>(cplane[p] + (size_t)(row * 8 + r) * uvls + x * 8 + 4 * q) = *reinterpret_cast<const uint32_t *>(&C[p][(1 + r) * CP + 4 + 4 * q]);
            }
            int16_t *gco = coeffs + m * coeff_stride;
            if (co16) { for (int i = lane; i < 96; i += 32) reinterpret_cast<uint4 *>(gco)[i] = reinterpret_cast<const uint4 *>(mb)[i]; }
            else      { for (int i = lane; i < 384; i += 32) reinterpret_cast<uint32_t *>(gco)[i] = reinterpret_cast<const uint32_t *>(mb)[i]; }
        }
        // publish: everything this macroblock wrote must be visible before the row below may read it
        __syncwarp();
        __threadfence();
        if (lane == 0) prog[row] = x + 1;
    }
}

// What h264_intra_kernel needs of its arguments (the header comment of ff_h264_intra_mb_batch_cuda): the records, nnzc and every coefficient
// row are fetched with 4-byte cp.async, the planes are read and written as words, and a macroblock fetches and writes back 768 coefficients
bool h264_intra_args_ok(const char *where, const void *mbs, const int16_t *coeffs, size_t coeff_stride, const uint8_t *nnzc, const uint8_t *luma,
                        const uint8_t *cb, const uint8_t *cr, int linesize, int uvlinesize, const uint32_t *progress)
{
    if (!mbs || !coeffs || !nnzc || !luma || !cb || !cr || !progress) { set_error_msg(where, "NULL argument"); return false; }
    if ((linesize & 3) || (uvlinesize & 3) || ((uintptr_t)luma & 3) || ((uintptr_t)cb & 3) || ((uintptr_t)cr & 3)) {
        set_error_msg(where, "planes and pitches must be 4-byte aligned"); return false;
    }
    if (((uintptr_t)mbs & 3) || ((uintptr_t)nnzc & 3) || ((uintptr_t)coeffs & 3) || (coeff_stride & 1)) {
        set_error_msg(where, "mbs, nnzc and coeffs must be 4-byte aligned and coeff_stride even"); return false;
    }
    if (coeff_stride < 768) { set_error_msg(where, "coeff_stride must be at least 768"); return false; }
    return true;
}

}  // namespace avb

using namespace avb;

extern "C" int ff_h264_intra_mb_batch_cuda(const FFH264IntraMB *mbs, int mb_w, int mb_h, int n_pictures, int16_t *coeffs,
                                           size_t coeff_stride, const uint8_t *nnzc, uint8_t *luma, uint8_t *cb, uint8_t *cr,
                                           int linesize, int uvlinesize, uint32_t *progress, void *stream)
{
    avb::enter();
    if (mb_w <= 0 || mb_h <= 0 || n_pictures <= 0) return 0;
    if (!h264_intra_args_ok("ff_h264_intra_mb_batch_cuda", mbs, coeffs, coeff_stride, nnzc, luma, cb, cr, linesize, uvlinesize, progress)) return -1;
    cudaStream_t st = (cudaStream_t)stream;
    const int rows = mb_h * n_pictures;
    AVB_CUDA(cudaMemsetAsync(progress, 0, sizeof(uint32_t) * rows, st), "ff_h264_intra_mb_batch_cuda");
    // a row only ever waits on the row above, which holds a lower ticket (taken by a CTA that started earlier), so any grid size makes progress
    static uint32_t *tickets = nullptr;                    // a small ring of counters: launches on different streams may overlap
    static unsigned next = 0;
    if (!tickets) AVB_CUDA(cudaMalloc(&tickets, 64 * sizeof(uint32_t)), "ff_h264_intra_mb_batch_cuda:tickets");
    uint32_t *ticket = tickets + (next++ % 64);
    AVB_CUDA(cudaMemsetAsync(ticket, 0, sizeof(uint32_t), st), "ff_h264_intra_mb_batch_cuda");
    h264_intra_kernel<<<rows, 32, 0, st>>>(mbs, mb_w, mb_h, coeffs, coeff_stride, nnzc, luma, cb, cr, linesize, uvlinesize, progress, ticket);
    return check_launch("ff_h264_intra_mb_batch_cuda");
}
