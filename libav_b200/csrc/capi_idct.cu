// libav_b200/csrc/capi_idct.cu -- C-ABI for the IDCTDSP / BlockDSP tables: batched device entry points,
// the host-buffer end-to-end call, per-block slot functions and the ff_*_init_cuda hooks.
#include "common.cuh"
#include "scratch.h"
#include "idct_dq.h"
#include "../../include/avdsp_b200.h"
#include <string.h>

namespace avb {
int launch_simple_idct(int mode, int16_t *blocks, uint8_t *frame, const uint32_t *dst_off, ptrdiff_t stride,
                       size_t n, int tiles_per_row, int clear, cudaStream_t st);
int launch_pixels_clamped(int mode, const int16_t *blocks, uint8_t *frame, const uint32_t *dst_off,
                          ptrdiff_t stride, size_t n, int tiles_per_row, cudaStream_t st);
int launch_clear_blocks(int16_t *blocks, size_t n_blocks, cudaStream_t st);
int launch_mpeg_dequant(int kind, const DqTables &t, const uint32_t *recs, int16_t *blocks, size_t n, cudaStream_t st);
int launch_mpeg_dequant_idct(int kind, const DqTables &t, const uint32_t *recs, int16_t *blocks, uint8_t *frame,
                             const uint32_t *dst_off, ptrdiff_t stride, size_t n, int tiles_per_row, int clear, cudaStream_t st);
int launch_mpeg_dequant_xvid_idct(int kind, const DqTables &t, const uint32_t *recs, int16_t *blocks, uint8_t *frame,
                                  const uint32_t *dst_off, ptrdiff_t stride, size_t n, int tiles_per_row, int clear, cudaStream_t st);
int launch_mpeg_dequant_faan_idct(int kind, const DqTables &t, const uint32_t *recs, int16_t *blocks, uint8_t *frame,
                                  const uint32_t *dst_off, ptrdiff_t stride, size_t n, int tiles_per_row, int clear, cudaStream_t st);
int launch_fill_blocks(uint8_t *frame, const uint32_t *dst_off, const uint8_t *value, ptrdiff_t stride, int h,
                       int w16, size_t n, cudaStream_t st);
}
using namespace avb;

extern "C" {

int ff_simple_idct_batch_cuda(int mode, int16_t *blocks, uint8_t *frame, const uint32_t *dst_off, ptrdiff_t stride,
                              size_t n, int tiles_per_row, int clear, void *stream)
{
    avb::enter();
    return launch_simple_idct(mode, blocks, frame, dst_off, stride, n, tiles_per_row, clear, (cudaStream_t)stream);
}
int ff_pixels_clamped_batch_cuda(int mode, const int16_t *blocks, uint8_t *frame, const uint32_t *dst_off,
                                 ptrdiff_t stride, size_t n, int tiles_per_row, void *stream)
{
    avb::enter();
    return launch_pixels_clamped(mode, blocks, frame, dst_off, stride, n, tiles_per_row, (cudaStream_t)stream);
}
static int dq_tables(const char *who, int kind, const FFMpegDequantTables *t, DqTables &d)
{
    if (!t || kind < 0 || kind > 6) { set_error_msg(who, "bad kind / tables"); return -1; }
    uint8_t seen[64] = { 0 };
    for (int i = 0; i < 64; i++) {
        if (t->permutated[i] > 63 || seen[t->permutated[i]]++) { set_error_msg(who, "permutated[] is not a permutation of 0..63"); return -1; }
        d.rank[t->permutated[i]] = (uint8_t)i;
        d.raster_end[i] = t->raster_end[i];
        d.intra[i] = t->intra_matrix[i]; d.inter[i] = t->inter_matrix[i];
    }
    d.alternate_scan = t->alternate_scan; d.h263_aic = t->h263_aic;
    return 0;
}
int ff_mpeg_dequant_batch_cuda(int kind, const FFMpegDequantTables *t, const FFMpegDequantBlock *recs, int16_t *blocks, size_t n,
                               void *stream)
{
    avb::enter();
    DqTables d;
    if (dq_tables("ff_mpeg_dequant_batch_cuda", kind, t, d)) return -1;
    return launch_mpeg_dequant(kind, d, reinterpret_cast<const uint32_t *>(recs), blocks, n, (cudaStream_t)stream);
}
int ff_mpeg_dequant_idct_batch_cuda(int kind, const FFMpegDequantTables *t, const FFMpegDequantBlock *recs, int16_t *blocks,
                                    uint8_t *frame, const uint32_t *dst_off, ptrdiff_t stride, size_t n, int tiles_per_row,
                                    int clear, void *stream)
{
    avb::enter();
    DqTables d;
    if (dq_tables("ff_mpeg_dequant_idct_batch_cuda", kind, t, d)) return -1;
    return launch_mpeg_dequant_idct(kind, d, reinterpret_cast<const uint32_t *>(recs), blocks, frame, dst_off, stride, n, tiles_per_row,
                                    clear, (cudaStream_t)stream);
}
int ff_mpeg_dequant_xvid_idct_batch_cuda(int kind, const FFMpegDequantTables *t, const FFMpegDequantBlock *recs, int16_t *blocks,
                                         uint8_t *frame, const uint32_t *dst_off, ptrdiff_t stride, size_t n, int tiles_per_row,
                                         int clear, void *stream)
{
    avb::enter();
    DqTables d;
    if (dq_tables("ff_mpeg_dequant_xvid_idct_batch_cuda", kind, t, d)) return -1;
    if (n && (((uintptr_t)blocks & 15) || (((uintptr_t)frame | (uintptr_t)stride) & 7))) {
        set_error_msg("ff_mpeg_dequant_xvid_idct_batch_cuda", "blocks must be 16-byte aligned, frame and stride multiples of 8");
        return -1;
    }
    return launch_mpeg_dequant_xvid_idct(kind, d, reinterpret_cast<const uint32_t *>(recs), blocks, frame, dst_off, stride, n, tiles_per_row,
                                         clear, (cudaStream_t)stream);
}
int ff_mpeg_dequant_faanidct_batch_cuda(int kind, const FFMpegDequantTables *t, const FFMpegDequantBlock *recs, int16_t *blocks,
                                        uint8_t *frame, const uint32_t *dst_off, ptrdiff_t stride, size_t n, int tiles_per_row,
                                        int clear, void *stream)
{
    avb::enter();
    DqTables d;
    if (dq_tables("ff_mpeg_dequant_faanidct_batch_cuda", kind, t, d)) return -1;
    if (n && (((uintptr_t)blocks & 15) || (((uintptr_t)frame | (uintptr_t)stride) & 7))) {
        set_error_msg("ff_mpeg_dequant_faanidct_batch_cuda", "blocks must be 16-byte aligned, frame and stride multiples of 8");
        return -1;
    }
    return launch_mpeg_dequant_faan_idct(kind, d, reinterpret_cast<const uint32_t *>(recs), blocks, frame, dst_off, stride, n, tiles_per_row,
                                         clear, (cudaStream_t)stream);
}
int ff_clear_blocks_batch_cuda(int16_t *blocks, size_t n_blocks, void *stream)
{
    avb::enter();
    return launch_clear_blocks(blocks, n_blocks, (cudaStream_t)stream);
}
int ff_fill_blocks_batch_cuda(uint8_t *frame, const uint32_t *dst_off, const uint8_t *value, ptrdiff_t stride, int h,
                              int w16, size_t n, void *stream)
{
    avb::enter();
    return launch_fill_blocks(frame, dst_off, value, stride, h, w16, n, (cudaStream_t)stream);
}

// ---- end-to-end with host buffers: chunked, three streams so H2D(k+1) / kernel(k) / D2H(k-1) overlap ----
int ff_simple_idct_batch_host_cuda(int mode, int16_t *blocks, uint8_t *frame, size_t frame_bytes,
                                   const uint32_t *dst_off, ptrdiff_t stride, size_t n, int tiles_per_row)
{
    avb::enter();
    if (n == 0) return 0;
    if (mode < 0 || mode > 2) { set_error_msg("simple_idct_batch_host", "bad mode"); return -1; }
    ScratchLock lk;
    Scratch &S = scratch();
    int16_t *d_blocks = (int16_t *)S.dev(0, n * 128);
    uint8_t *d_frame = mode == 2 ? nullptr : (uint8_t *)S.dev(1, frame_bytes);
    uint32_t *d_off = (mode != 2 && dst_off) ? (uint32_t *)S.dev(2, n * 4) : nullptr;
    if (!d_blocks || (mode != 2 && !d_frame) || (mode != 2 && dst_off && !d_off)) return -1;
    cudaStream_t *st = S.streams();
    if (!st) return -1;

    // Only the pixels that blocks address may change in the caller's frame.  Banded (raster-of-tiles) addressing
    // lets each chunk own whole tile rows: its band is downloaded with a 2-D copy limited to the tile columns (and,
    // for a ragged last tile row, to the tiles that exist).  With explicit offsets the touched set is arbitrary, so
    // the frame is uploaded first and downloaded whole.
    const bool banded = mode != 2 && !dst_off && tiles_per_row > 0 && stride >= (ptrdiff_t)tiles_per_row * 8;
    size_t chunk = 1 << 16;
    if (banded) { size_t rows = chunk / tiles_per_row; if (rows < 1) rows = 1; chunk = rows * tiles_per_row; }
    if (mode != 2 && !banded) AVB_CUDA(cudaMemcpyAsync(d_frame, frame, frame_bytes, cudaMemcpyHostToDevice, st[0]), "idct_host:h2d frame");
    if (d_off) AVB_CUDA(cudaMemcpyAsync(d_off, dst_off, n * 4, cudaMemcpyHostToDevice, st[0]), "idct_host:h2d off");
    if ((mode != 2 && !banded) || d_off) {
        AVB_CUDA(cudaEventRecord(S.event(0), st[0]), "idct_host");
        for (int k = 1; k < 3; k++) AVB_CUDA(cudaStreamWaitEvent(st[k], S.event(0), 0), "idct_host");
    }
    int k = 0;
    for (size_t lo = 0; lo < n; lo += chunk, k = (k + 1) % 3) {
        size_t cnt = n - lo < chunk ? n - lo : chunk;
        cudaStream_t s = st[k];
        AVB_CUDA(cudaMemcpyAsync(d_blocks + lo * 64, blocks + lo * 64, cnt * 128, cudaMemcpyHostToDevice, s), "idct_host:h2d blocks");
        if (banded) {
            const size_t row0 = lo / tiles_per_row, full = cnt / tiles_per_row, rem = cnt % tiles_per_row;
            const size_t band_off = row0 * 8 * (size_t)stride, wfull = (size_t)tiles_per_row * 8;
            uint8_t *hb = frame + band_off, *db = d_frame + band_off;
            if (mode == 1) {
                if (full) AVB_CUDA(cudaMemcpy2DAsync(db, stride, hb, stride, wfull, full * 8, cudaMemcpyHostToDevice, s), "idct_host:h2d band");
                if (rem) AVB_CUDA(cudaMemcpy2DAsync(db + full * 8 * stride, stride, hb + full * 8 * stride, stride, rem * 8, 8, cudaMemcpyHostToDevice, s), "idct_host:h2d band");
            }
            if (launch_simple_idct(mode, d_blocks + lo * 64, db, nullptr, stride, cnt, tiles_per_row, 0, s)) return -1;
            if (full) AVB_CUDA(cudaMemcpy2DAsync(hb, stride, db, stride, wfull, full * 8, cudaMemcpyDeviceToHost, s), "idct_host:d2h band");
            if (rem) AVB_CUDA(cudaMemcpy2DAsync(hb + full * 8 * stride, stride, db + full * 8 * stride, stride, rem * 8, 8, cudaMemcpyDeviceToHost, s), "idct_host:d2h band");
        } else {
            if (launch_simple_idct(mode, d_blocks + lo * 64, d_frame, d_off ? d_off + lo : nullptr, stride, cnt, tiles_per_row, 0, s)) return -1;
            if (mode == 2) AVB_CUDA(cudaMemcpyAsync(blocks + lo * 64, d_blocks + lo * 64, cnt * 128, cudaMemcpyDeviceToHost, s), "idct_host:d2h blocks");
        }
    }
    for (int i = 0; i < 3; i++) AVB_CUDA(cudaStreamSynchronize(st[i]), "idct_host:sync");
    if (mode != 2 && !banded) {
        AVB_CUDA(cudaMemcpyAsync(frame, d_frame, frame_bytes, cudaMemcpyDeviceToHost, st[0]), "idct_host:d2h frame");
        AVB_CUDA(cudaStreamSynchronize(st[0]), "idct_host:sync");
    }
    return 0;
}

}  // extern "C"

// ---------------------------------------------------------------------------------------------------
// Slot functions: same signatures as the C slots, HOST pointers, one block per call.
// ---------------------------------------------------------------------------------------------------
namespace {

// copy an 8-row x `w`-byte host region with arbitrary (possibly negative) stride to/from a packed buffer
void gather_rows(uint8_t *packed, const uint8_t *src, ptrdiff_t stride, int w, int h)
{ for (int y = 0; y < h; y++) memcpy(packed + y * w, src + y * stride, w); }
void scatter_rows(uint8_t *dst, ptrdiff_t stride, const uint8_t *packed, int w, int h)
{ for (int y = 0; y < h; y++) memcpy(dst + y * stride, packed + y * w, w); }

// one block through the batched kernel: staging = [128 B block][64 B pixels] pinned + device mirrors
int slot_block_op(int family, int mode, int16_t *block, uint8_t *dest, ptrdiff_t line_size)
{
    ScratchLock lk;
    Scratch &S = scratch();
    uint8_t *h = (uint8_t *)S.pinned(256);
    uint8_t *d = (uint8_t *)S.dev(3, 256);
    cudaStream_t *st = S.streams();
    if (!h || !d || !st) return -1;
    cudaStream_t s = st[0];
    bool reads_dest = dest && ((family == 0 && mode == 1) || (family == 1 && mode == 2));
    memcpy(h, block, 128);
    if (reads_dest) gather_rows(h + 128, dest, line_size, 8, 8);
    AVB_CUDA(cudaMemcpyAsync(d, h, reads_dest ? 192 : 128, cudaMemcpyHostToDevice, s), "slot:h2d");
    int rc = family == 0 ? launch_simple_idct(mode, (int16_t *)d, d + 128, nullptr, 8, 1, 1, 0, s)
                         : launch_pixels_clamped(mode, (const int16_t *)d, d + 128, nullptr, 8, 1, 1, s);
    if (rc) return -1;
    AVB_CUDA(cudaMemcpyAsync(h, d, 192, cudaMemcpyDeviceToHost, s), "slot:d2h");
    AVB_CUDA(cudaStreamSynchronize(s), "slot:sync");
    if (family == 0 && mode == 2) memcpy(block, h, 128);
    else scatter_rows(dest, line_size, h + 128, 8, 8);
    return 0;
}

void slot_idct_put(uint8_t *dest, ptrdiff_t ls, int16_t *block) { slot_block_op(0, 0, block, dest, ls); }
void slot_idct_add(uint8_t *dest, ptrdiff_t ls, int16_t *block) { slot_block_op(0, 1, block, dest, ls); }
void slot_idct(int16_t *block) { slot_block_op(0, 2, block, nullptr, 0); }
void slot_put_pixels_clamped(const int16_t *b, uint8_t *AVB_RESTRICT p, ptrdiff_t ls) { slot_block_op(1, 0, (int16_t *)b, p, ls); }
void slot_put_signed_pixels_clamped(const int16_t *b, uint8_t *AVB_RESTRICT p, ptrdiff_t ls) { slot_block_op(1, 1, (int16_t *)b, p, ls); }
void slot_add_pixels_clamped(const int16_t *b, uint8_t *AVB_RESTRICT p, ptrdiff_t ls) { slot_block_op(1, 2, (int16_t *)b, p, ls); }

int slot_clear(int16_t *blocks, int nblk)
{
    ScratchLock lk;
    Scratch &S = scratch();
    size_t bytes = (size_t)nblk * 128;
    uint8_t *h = (uint8_t *)S.pinned(1024);
    uint8_t *d = (uint8_t *)S.dev(3, 1024);
    cudaStream_t *st = S.streams();
    if (!h || !d || !st) return -1;
    // the block contents are irrelevant to the result, but the op runs on the device all the same
    if (launch_clear_blocks((int16_t *)d, nblk, st[0])) return -1;
    AVB_CUDA(cudaMemcpyAsync(h, d, bytes, cudaMemcpyDeviceToHost, st[0]), "slot_clear:d2h");
    AVB_CUDA(cudaStreamSynchronize(st[0]), "slot_clear:sync");
    memcpy(blocks, h, bytes);
    return 0;
}
void slot_clear_block(int16_t *b) { slot_clear(b, 1); }
void slot_clear_blocks(int16_t *b) { slot_clear(b, 6); }

void slot_fill(uint8_t *block, uint8_t value, ptrdiff_t ls, int h, int w16)
{
    ScratchLock lk;
    Scratch &S = scratch();
    int w = w16 ? 16 : 8;
    uint8_t *hp = (uint8_t *)S.pinned(1024);
    uint8_t *d = (uint8_t *)S.dev(3, 1024);
    cudaStream_t *st = S.streams();
    if (!hp || !d || !st || h > 32) return;
    // device layout: [0,512) pixel rows (stride w) | 512: uint32 offset | 516: value
    uint32_t off = 0;
    memcpy(hp + 512, &off, 4); hp[516] = value;
    if (cudaMemcpyAsync(d + 512, hp + 512, 8, cudaMemcpyHostToDevice, st[0]) != cudaSuccess) { set_error("slot_fill", cudaGetLastError()); return; }
    if (launch_fill_blocks(d, (const uint32_t *)(d + 512), d + 516, w, h, w16, 1, st[0])) return;
    if (cudaMemcpyAsync(hp, d, (size_t)w * h, cudaMemcpyDeviceToHost, st[0]) != cudaSuccess || cudaStreamSynchronize(st[0]) != cudaSuccess) { set_error("slot_fill", cudaGetLastError()); return; }
    scatter_rows(block, ls, hp, w, h);
}
void slot_fill16(uint8_t *b, uint8_t v, ptrdiff_t ls, int h) { slot_fill(b, v, ls, h, 1); }
void slot_fill8(uint8_t *b, uint8_t v, ptrdiff_t ls, int h) { slot_fill(b, v, ls, h, 0); }

}  // namespace

namespace avb { void idct10_install(IDCTDSPContext *c); }      // idct10.cu
namespace avb { void faan_idct_install(IDCTDSPContext *c); }   // faan_idct.cu

extern "C" {

void ff_idctdsp_init_cuda(IDCTDSPContext *c, int idct_algo, int bits_per_raw_sample, unsigned high_bit_depth)
{
    avb::enter();
    if (bits_per_raw_sample == 10) {                                    // idctdsp.c:151-155: the 10-bit simple IDCT whatever idct_algo says;
        idct10_install(c);                                              // the three pixel-clamp entries are the 8-bit functions at every depth (:175-177)
        c->put_pixels_clamped        = slot_put_pixels_clamped;
        c->put_signed_pixels_clamped = slot_put_signed_pixels_clamped;
        c->add_pixels_clamped        = slot_add_pixels_clamped;
        return;
    }
    if (high_bit_depth || bits_per_raw_sample > 8) return;              // 9 / 12-bit ...: the reference falls through to its 8-bit table there; not taken over
    c->put_pixels_clamped        = slot_put_pixels_clamped;
    c->put_signed_pixels_clamped = slot_put_signed_pixels_clamped;
    c->add_pixels_clamped        = slot_add_pixels_clamped;
    if (idct_algo == AVB_FF_IDCT_AUTO || idct_algo == AVB_FF_IDCT_SIMPLE) {
        c->idct      = slot_idct;
        c->idct_put  = slot_idct_put;
        c->idct_add  = slot_idct_add;
        c->perm_type = FF_IDCT_PERM_NONE;          // same as the C simple IDCT, libavcodec/idctdsp.c:172
        // ff_idctdsp_init() calls ff_init_scantable_permutation() after the arch hooks; keep the table
        // consistent for callers that invoke the hook on its own.
        for (int i = 0; i < 64; i++) c->idct_permutation[i] = (uint8_t)i;
    } else if (idct_algo == AVB_FF_IDCT_FAAN) {
        faan_idct_install(c);                      // idctdsp.c:162-166
    }
}

void ff_blockdsp_init_cuda(BlockDSPContext *c)
{
    avb::enter();
    c->clear_block       = slot_clear_block;
    c->clear_blocks      = slot_clear_blocks;
    c->fill_block_tab[0] = slot_fill16;
    c->fill_block_tab[1] = slot_fill8;
}

}  // extern "C"
