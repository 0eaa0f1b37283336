/*
 * include/avdsp_b200.h -- C ABI of libavdsp_b200.so, the sm_90a (H100) back-end for libav's per-block DSP
 * tables and the libswscale scaler.  Plain C: pointers and sizes only, no C++/torch types.
 *
 * Three layers, all in this one header:
 *   1. runtime      avb200_*            device selection, sticky error, memory/stream helpers
 *   2. batched ops  ff_*_batch_cuda     DEVICE pointers, asynchronous on `stream` (a cudaStream_t passed
 *                                       as void *, NULL = default stream).  These are the fast path:
 *                                       thousands of blocks / whole frames per launch.
 *   3. table hooks  ff_*_init_cuda      fill the reference's own function-pointer tables (structs in
 *                                       avdsp_b200_tables.h are layout-identical to the reference's) with
 *                                       slot functions that take HOST pointers exactly like the C slots
 *                                       (one block per call: upload, launch, download, sync).  They exist
 *                                       so the CUDA path drops in behind ff_*dsp_init()'s arch dispatch
 *                                       (libavcodec/idctdsp.c:183-188 etc.); they are for plumbing and
 *                                       parity, not speed.
 * Error convention: the reference slots return void (SURVEY 8b).  Every entry point here that can fail
 * returns 0 / -1 and records a message (avb200_last_error()); slot functions record it too.  The first CUDA FAILURE sticks until
 * avb200_clear_error(); a REFUSAL (a request this library does not take over: the caller keeps its C path) is held only until a
 * failure arrives, so routine refusals never hide a real fault.  There is NO CPU fallback: without an H100 every call fails loudly.
 */
#ifndef AVDSP_B200_H
#define AVDSP_B200_H

#include <stddef.h>
#include <stdint.h>
#include "avdsp_b200_tables.h"

#ifdef __cplusplus
extern "C" {
#endif

/* ------------------------------------------------------------------ 1. runtime ------------------- */
int         avb200_device_count(void);
int         avb200_init(int device);              /* cudaSetDevice + context warm-up; -1 if no sm_100 GPU */
const char *avb200_last_error(void);              /* "" when no error is pending */
void        avb200_clear_error(void);
void        avb200_set_log_callback(void (*cb)(int av_log_level, const char *msg)); /* av_log-style sink */
void        avb200_set_tuning(const char *key, int value);   /* test knobs that force a fallback kernel the library picks for other
                                                               inputs: sws_general_variant, mc_variant, residual_variant, idct_tma
                                                               (0 = the default); unknown keys are ignored */
void       *avb200_malloc(size_t bytes);          /* device memory */
void        avb200_free(void *dptr);
void       *avb200_host_alloc(size_t bytes);      /* pinned host memory */
void        avb200_host_free(void *hptr);
int         avb200_host_register(void *hptr, size_t bytes);
int         avb200_host_unregister(void *hptr);
int         avb200_memcpy_h2d(void *dst, const void *src, size_t bytes, void *stream);
int         avb200_memcpy_d2h(void *dst, const void *src, size_t bytes, void *stream);
int         avb200_memcpy2d_h2d(void *dst, size_t dpitch, const void *src, size_t spitch, size_t width, size_t height, void *stream);
int         avb200_memcpy2d_d2h(void *dst, size_t dpitch, const void *src, size_t spitch, size_t width, size_t height, void *stream);
int         avb200_memset(void *dst, int value, size_t bytes, void *stream);
void       *avb200_stream_create(void);
void        avb200_stream_destroy(void *stream);
int         avb200_stream_sync(void *stream);
int         avb200_device_sync(void);
void       *avb200_event_create(void);
void        avb200_event_destroy(void *ev);
int         avb200_event_record(void *ev, void *stream);
int         avb200_event_sync(void *ev);
float       avb200_event_elapsed_ms(void *start, void *stop);

/* ------------------------------------------------------------------ 2. batched ops --------------- */
/*
 * Destination addressing shared by the 8x8 block ops: block i is written at
 *     frame + dst_off[i]                                  when dst_off != NULL (byte offsets), else at
 *     frame + (i / tiles_per_row) * 8 * stride + (i % tiles_per_row) * 8   (raster of 8x8 tiles).
 * `blocks` is n * 64 int16_t, block-major, row-major inside a block, 16-byte aligned -- the layout the
 * reference's callers hand to idsp.idct_put (libavcodec/mpegvideo.c:1401-1427).
 */

/* IDCTDSPContext.idct_put / idct_add / idct with idct_algo = FF_IDCT_SIMPLE
 * (libavcodec/simple_idct_template.c:289-326, selected at libavcodec/idctdsp.c:168-173).
 * mode 0 = put, 1 = add, 2 = in-place int16 (frame/dst_off/stride ignored).
 * clear != 0 additionally zeroes each coefficient block (fused BlockDSPContext.clear_block,
 * libavcodec/blockdsp.c:29-32); otherwise `blocks` is left untouched (the reference leaves its
 * row-pass intermediate there; callers must not rely on either). */
int ff_simple_idct_batch_cuda(int mode, int16_t *blocks, uint8_t *frame, const uint32_t *dst_off,
                              ptrdiff_t stride, size_t n, int tiles_per_row, int clear, void *stream);

/* IDCTDSPContext.put_pixels_clamped / put_signed_pixels_clamped / add_pixels_clamped
 * (libavcodec/idctdsp.c:85-145).  mode 0 / 1 / 2. */
int ff_pixels_clamped_batch_cuda(int mode, const int16_t *blocks, uint8_t *frame, const uint32_t *dst_off,
                                 ptrdiff_t stride, size_t n, int tiles_per_row, void *stream);

/* ff_simple_idct_put_10 / _add_10 / _10 (libavcodec/simple_idct_template.c, BIT_DEPTH 10; idctdsp.c:151-155) over n blocks: mode 0 put, 1 add,
 * 2 in place; block i -> the 8 x 8 16-bit samples at frame + dst_off[i] (bytes), rows `stride` bytes apart.  The blocks are left as the C
 * functions leave them.  Functional path for 10-bit content (thread per block), not tuned like the 8-bit kernel. */
int ff_simple_idct10_batch_cuda(int mode, int16_t *blocks, uint8_t *frame, const uint32_t *dst_off, ptrdiff_t stride, size_t n, void *stream);

/* ---- ProRes (libavcodec/proresdsp.c, proresdec.c) ---------------------------------------------------------------------------------------
 * prores_idct_put_c over n blocks: block i is multiplied by the 64 int16 of qmats + 64 * qmat_idx[i] (matrix 0 for every block when
 * qmat_idx is NULL; products wrap to int16), transformed by ff_prores_idct and written as av_clip(v + 512, 4, 1019) into the 8 x 8 16-bit
 * samples at frame + dst_off[i] (bytes), rows `stride` bytes apart.  Each block is left as the C function leaves it: the column pass's
 * int16 results.  Device pointers, on `stream`, without synchronising.  Blocks and qmats 16-byte aligned with a stride that is a multiple
 * of 16 run the staged kernel, anything else a thread-per-block kernel.  Returns -1 for NULL pointers with n > 0 or an odd stride. */
int ff_prores_idct_put_batch_cuda(int16_t *blocks, uint8_t *frame, const uint32_t *dst_off, ptrdiff_t stride, const int16_t *qmats,
                                  const uint32_t *qmat_idx, size_t n, void *stream);

/* One slice of a ProRes picture as decode_picture / decode_slice see it (device memory).  sf: the slice's scale factor after
 * decode_slice's mapping (1..512); first_block: the slice's first coefficient block in FFProresPictureWork.blocks. */
typedef struct FFProresSlice {
    uint32_t first_block;
    uint16_t sf;
    uint16_t reserved;
} FFProresSlice;
/* One ProRes picture (a frame, or one field of an interlaced frame) whose slices were entropy-decoded but not transformed.  The
 * coefficient buffer is in the decoder's order: per slice (raster order, as decode_picture numbers them), its luma blocks, then U, then V,
 * each plane in decode_slice_plane's order (luma TL TR BL BR per macroblock; 4:2:2 chroma top, bottom; 4:4:4 chroma TL BL TR BR).
 * The call derives each block's destination and scaled matrix (int16_t)(qmat[i] * sf) on the device.  Blocks inside the buffer that no
 * slice covers are skipped. */
typedef struct FFProresPictureWork {
    uint8_t *data[3];            /* device: y, u, v as decode_slice computes them (a field's second picture starts one frame line down) */
    int linesize[3];             /* bytes between the picture's lines (doubled for a field), even and > 0; at least the width of whole
                                  * macroblocks (32 * mb_width bytes for luma and 4:4:4 chroma, 16 * mb_width for 4:2:2 chroma).  The call
                                  * sees only this linesize: for a field it cannot tell a frame buffer narrower than whole macroblocks
                                  * (whose two fields' rows then overlap) from a wide one, so the caller guarantees the frame linesize */
    int mb_rows[3];              /* 16-line rows at linesize each plane buffer holds from data[p]: at least mb_height */
    int mb_width, mb_height;     /* ctx->num_x_mbs, ctx->num_y_mbs (macroblock rows of this picture) */
    int slice_width_factor;      /* 0..3 */
    int chroma_format;           /* ctx->chroma_factor: 2 = 4:2:2, 3 = 4:4:4 */
    uint8_t qmat_luma[64], qmat_chroma[64];     /* ctx->qmat_luma / qmat_chroma (FF_IDCT_PERM_NONE order) */
    const FFProresSlice *slices; /* device, n_slices entries */
    int n_slices;                /* must be the picture's slice count, mb_height * slices per row */
    const int16_t *blocks;       /* device, n_blocks * 64 coefficients, left unchanged */
    size_t n_blocks;
} FFProresPictureWork;
/* The flush point of a ProRes decoder: the inverse quantisation, IDCT and store of n pictures, on `stream`, without synchronising; nothing
 * else is read or written (no alpha plane).  Every picture is checked before anything is launched; -1 for a NULL array, a chroma_format
 * other than 2 / 3, slice_width_factor > 3, macroblock dimensions outside 1..8192, a NULL or odd plane pointer or linesize, planes too
 * small for whole macroblocks (width or mb_rows), a slice count that does not cover the picture, or NULL slices / blocks. */
int ff_prores_decode_pictures_cuda(const FFProresPictureWork *pictures /* host array */, int n, void *stream);

/* ---- ProRes decoder, whole packets (libavcodec/proresdec.c: decode_frame) ---------------------------------------------------------------
 * Semantics:
 *  1. Each packet decodes as a fresh decoder context decodes it.  (A reference context carries nothing that changes the samples from one
 *     packet to the next: decode_frame_header rewrites qmat_luma / qmat_chroma for every frame and decode_picture_header resets each
 *     slice's prev_slice_sf, so this call has no context.)
 *  2. A slice's errors never abort the frame (avctx->execute ignores decode_slice's return value).  Within a slice: a slice under 6 bytes,
 *     or with plane sizes that do not fit it or a header size under 6, writes nothing; a plane whose AC decoding fails is not written, and
 *     neither is any plane after it; alpha is written only when Y, U and V all decoded and the slice has alpha bytes.
 *  3. Each slice plane is read with the reference's checked long reader: past the plane's end it sees the packet's following bytes, past
 *     the packet's end zeros (the packet's padding); the position stops at the plane's bits + 8; get_bits_left and the MAX_PADDING test are
 *     relative to the plane.
 *  4. decode_vlc_codeword's exp-Golomb branch shifts by 32 - len with len up to 68 (a run of zero bits, as on a zero-filled plane, whose
 *     DC decoding has no end guard).  A negative count is undefined in C; the reference as compiled for x86-64 shifts by the count modulo
 *     32, and so does this call.
 *  5. Arithmetic wraps as the compiled reference's does: DC (prev_dc, delta) and AC levels are truncated to int16, a code read as a
 *     negative run or level ends the plane with an error, and each scaled matrix entry is (int16_t)(qmat * sf).
 *  6. Header oddities decode as the reference decodes them: a frame header hdr_size below 20 still reads bytes 8..19; a first
 *     pic_data_size of 0 decodes the same picture data again into the second field; a pic_data_size of 2^31 or more is an error before its
 *     picture is decoded; a second picture header that fails leaves the first field written (FFProresFrameInfo.result).
 * Refusals beyond the reference's own (each -1 with a message): a packet the probe does not return 0 for (no frame exists to write); a zero
 * width or height (get_buffer refuses such a frame); NULL or odd planes; linesizes that are not even, not positive, or narrower than whole
 * macroblocks (32 bytes per macroblock for luma, alpha and 4:4:4 chroma, 16 for 4:2:2 chroma); planes with fewer than
 * FFProresFrameInfo.lines lines; a missing alpha plane for a format with alpha; a NULL device packet; a workspace smaller than
 * ff_prores_decode_workspace_cuda returns, or not 16-byte aligned (its coefficient blocks are zeroed and read 16 bytes at a time). */
#define FF_PRORES_PIX_FMT_YUV422P10  66      /* AV_PIX_FMT_YUV422P10 (little-endian) */
#define FF_PRORES_PIX_FMT_YUV444P10  70      /* AV_PIX_FMT_YUV444P10 */
#define FF_PRORES_PIX_FMT_YUVA422P10 92      /* AV_PIX_FMT_YUVA422P10 */
#define FF_PRORES_PIX_FMT_YUVA444P10 94      /* AV_PIX_FMT_YUVA444P10 */
/* What decode_frame sets up for a packet, and what it returns. */
typedef struct FFProresFrameInfo {
    int pix_fmt;                 /* FF_PRORES_PIX_FMT_* */
    int interlaced_frame, top_field_first;
    int color_primaries, color_trc, colorspace;  /* the frame header's three colour bytes */
    int lines;                   /* lines each plane must hold: num_y_mbs * 16 << interlaced_frame (the decoder writes whole macroblocks, in
                                  * width and in height) */
    int pictures;                /* pictures the decoder decodes: 0, 1 or 2 (fewer than the frame's when a picture header fails) */
    int result;                  /* decode_frame's return value: the packet size, or AVERROR_INVALIDDATA after a failing picture header */
} FFProresFrameInfo;
/* decode_frame's checks up to get_buffer (the frame atom, decode_frame_header) on the host, and both decode_picture_header calls' (the
 * slice-table sums included); nothing is launched.  width / height: the caller's avctx dimensions, which the header must match.  Returns
 * 0, the AVERROR_INVALIDDATA the reference returns before get_buffer, or -1 with a message for a refusal listed above.  A decoder calls it
 * in place of decode_frame_header, then get_buffer, then ff_prores_decode_frames_cuda, and returns info.result. */
int ff_prores_probe_cuda(const uint8_t *pkt_host, int size, int width, int height, FFProresFrameInfo *info);
/* One packet for ff_prores_decode_frames_cuda. */
typedef struct FFProresDecodeWork {
    const uint8_t *pkt_host;     /* the packet on the host, for its headers */
    const uint8_t *pkt;          /* the same bytes on the device */
    int size;
    int width, height;           /* avctx->width / height */
    uint8_t *data[4];            /* device planes of 16-bit samples (even addresses): y, u, v, and alpha for the yuva formats */
    int linesize[4];             /* bytes between the frame's lines: even, positive, at least the width of whole macroblocks */
    int lines[4];                /* lines each plane holds: at least FFProresFrameInfo.lines */
} FFProresDecodeWork;
/* Bytes of device workspace ff_prores_decode_frames_cuda needs for these packets (host only, nothing launched); 0 for a batch with a packet
 * or plane the decode call refuses. */
size_t ff_prores_decode_workspace_cuda(const FFProresDecodeWork *works /* host array */, int n);
/* decode_frame for n packets on `stream`, without synchronising: every sample the reference decoder writes is written with its value (the
 * alpha plane, and the pictures before a failing second picture header, included), and nothing else.  Every packet is checked (the probe's
 * checks, then the planes) before anything is launched; -1 with a message for a refusal listed above. */
int ff_prores_decode_frames_cuda(const FFProresDecodeWork *works /* host array */, int n, void *workspace, size_t workspace_bytes, void *stream);

/* ---- ProRes encoder (libavcodec/proresenc.c) --------------------------------------------------------------------------------------------
 * One frame for ff_prores_encode_frames_cuda: the source planes and the encoder's options, as encode_init / encode_frame take them. */
typedef struct FFProresEncodeWork {
    const uint8_t *data[4];      /* device: y, u, v (and alpha for yuva444p10) planes of 16-bit samples in 0..1023, even addresses */
    int linesize[4];             /* bytes between lines, even, at least the plane's width in bytes (4:2:2 chroma: (width + 1) / 2 samples) */
    int width, height;           /* 1..65535; interlaced heights 1 and 32k + 1 are refused (a field's last macroblock row has no lines) */
    int pix_fmt;                 /* 0 yuv422p10, 1 yuv444p10, 2 yuva444p10 */
    int interlaced;              /* 0 progressive, 1 top field first, 2 bottom field first (AV_CODEC_FLAG_INTERLACED_DCT + top_field_first) */
    int profile;                 /* 0..4: proxy, LT, standard, HQ, 4444 (the encoder's "profile" option) */
    int mbs_per_slice;           /* 1, 2, 4, 8 */
    int bits_per_mb;             /* 0 = from the profile's table for the frame size, else 128..8192 (ignored under force_quant) */
    int quant_sel;               /* -1 = the profile's matrix, 0..4 (the "quant_mat" option; 4 = default, not written to the header) */
    int alpha_bits;              /* 0, 8, 16; only read for yuva444p10 */
    int force_quant;             /* 0 = rate control, 1..64 = one quantiser for every slice (global_quality / FF_QP2LAMBDA) */
    char vendor[4];              /* four non-zero bytes */
    uint8_t color_primaries, color_trc, colorspace;
    uint8_t *out;                /* device packet buffer */
    size_t out_capacity;
    int32_t *out_size;           /* device, 4-byte aligned: the packet's size, or -(size needed) with out untouched when it does not fit */
} FFProresEncodeWork;
/* Bytes of device workspace ff_prores_encode_frames_cuda needs for these frames (host only, nothing launched); 0 for a refused batch. */
size_t ff_prores_encode_workspace_cuda(const FFProresEncodeWork *frames /* host array */, int n);
/* encode_frame for n frames on `stream`, without synchronising: each packet is the reference encoder's for the same frame and options, byte
 * for byte, with find_quant_thread's rate control (or force_quant) and every slice coded on the device.  Every frame is checked before
 * anything is launched; -1 with a message for what encode_init refuses (pix_fmt, interlaced, profile or quant_sel out of range,
 * mbs_per_slice not 1 / 2 / 4 / 8, alpha_bits not 0 / 8 / 16, bits_per_mb in 1..127 without force_quant or above 8192, force_quant outside
 * 0..64, a vendor ID with a zero byte), NULL or odd planes, odd or narrow linesizes, sizes the headers cannot hold (width or height outside
 * 1..65535, more than 65535 slices per picture), interlaced heights 1 and 32k + 1, a NULL out / out_size, and a workspace smaller than
 * ff_prores_encode_workspace_cuda returns. */
int ff_prores_encode_frames_cuda(const FFProresEncodeWork *frames /* host array */, int n, void *workspace, size_t workspace_bytes, void *stream);

/* ---- VC-3 / DNxHD encoder (libavcodec/dnxhdenc.c) -----------------------------------------------------------------------------------------
 * CIDEntry (libavcodec/dnxhddata.h:28-42), field for field: the encoder's ctx->cid_table.  The library builds its device VLC, run and
 * weight tables from the entry, caches them by the entry's host address and rebuilds them when a checksum of the arrays changes. */
typedef struct FFDnxhdCidEntry {
    int cid;
    unsigned int width, height;
    int interlaced;
    unsigned int frame_size;
    unsigned int coding_unit_size;
    int index_bits;
    int bit_depth;
    const uint8_t *luma_weight, *chroma_weight;
    const uint8_t *dc_codes, *dc_bits;
    const uint16_t *ac_codes;
    const uint8_t *ac_bits, *ac_level;
    const uint8_t *ac_run_flag, *ac_index_flag;
    const uint16_t *run_codes;
    const uint8_t *run_bits, *run;
    int bit_rates[5];
} FFDnxhdCidEntry;
/* The rate-control state that DNXHDEncContext carries from field to field and frame to frame; a new encoder starts at { 1, 2 << 10 }
 * (dnxhd_init_rc).  The fast rate control needs qscale in 1..qmax - 1, where the encoder leaves it; a frame that finds it elsewhere fails
 * with EINVAL.  After a failure the state is what the reference leaves: the last qscale find_qscale tried, lambda untouched by RD. */
typedef struct FFDnxhdRcState { uint32_t qscale, lambda; } FFDnxhdRcState;
/* One frame for ff_dnxhd_encode_frames_cuda, as dnxhd_encode_picture takes it. */
typedef struct FFDnxhdEncodeWork {
    const uint8_t *data[3];      /* device planes: yuv422p (8-bit samples) or yuv422p10 (16-bit samples in 0..1023, even addresses).  For
                                  * 1080-line 10-bit CIDs the luma plane must have 1088 readable lines: the variance pass of the fast rate
                                  * control reads all 16 lines of the last macroblock row, as dnxhd_mb_var_thread does, and those 8 lines
                                  * change the packet */
    int linesize[3];             /* bytes between lines, positive; even at 10 bit; at least the plane's width in bytes */
    const FFDnxhdCidEntry *cid_table;  /* host: the entry the encoder chose (ff_dnxhd_cid_table[i]); size, interlacing, bit depth */
    int interlaced;              /* 0 progressive, 1 top field first, 2 bottom field first (cur_field of dnxhd_load_picture); must match
                                  * cid_table->interlaced */
    int dct_algo;                /* 8 bit only: FF_DCT_FASTINT (1) ifast, FF_DCT_FAAN (6) FAAN, anything else islow */
    int mb_decision;             /* FF_MB_DECISION_RD (2): dnxhd_encode_rdo; anything else: dnxhd_encode_fast */
    int qmax;                    /* 2..69 */
    int nitris_compat;           /* 0 or 1 (min_padding 1600) */
    FFDnxhdRcState *state;       /* device; frames sharing a pointer are encoded in array order, as one context encodes them */
    uint8_t *out;                /* device, 4-byte aligned: cid_table->frame_size bytes are written, never more */
    size_t out_capacity;         /* at least cid_table->frame_size */
    int32_t *out_info;           /* device: [0] the packet size (frame_size) or AVERROR(EINVAL) when rate control cannot fit the picture
                                  * (the packet bytes are then unspecified), [1] qscale * FF_QP2LAMBDA, the quality side data (with
                                  * FF_MB_DECISION_RD qscale is qmax - 1, where dnxhd_encode_rdo's table loop leaves ctx->qscale) */
} FFDnxhdEncodeWork;
/* Bytes of device workspace ff_dnxhd_encode_frames_cuda needs for these frames (host only, nothing launched); 0 for a refused batch. */
size_t ff_dnxhd_encode_workspace_cuda(const FFDnxhdEncodeWork *frames /* host array */, int n);
/* dnxhd_encode_picture for n frames on `stream`, without synchronising: each packet is the reference encoder's for the same frame, options
 * and state, byte for byte, and each state is left as the encoder leaves its context, after a rate-control failure too.  Every frame is
 * checked before anything is launched; -1 with a message for NULL or odd planes and linesizes, linesizes narrower than the plane, a CID
 * entry with a bit depth other than 8 / 10 or one dnxhd_init_vlc would reject (a level without a code, a run of 0 or past 62, a run listed
 * twice), interlacing that does not match the entry, qmax outside 2..69, nitris_compat not 0 / 1, out_capacity below frame_size, a NULL or
 * misaligned out, a NULL state or out_info, and a workspace smaller than ff_dnxhd_encode_workspace_cuda returns. */
int ff_dnxhd_encode_frames_cuda(const FFDnxhdEncodeWork *frames /* host array */, int n, void *workspace, size_t workspace_bytes, void *stream);

/* ---- VC-3 / DNxHD decoder (libavcodec/dnxhddec.c) -----------------------------------------------------------------------------------------
 * Semantics:
 *  1. Each packet decodes as a fresh decoder context decodes it.  (A reference context caches its VLCs per CID and never clears is_444, so
 *     within one context a bit-depth or 4:4:4 change under the same CID reuses stale tables; this call has no context.)
 *  2. Bits at and past `size` read as zero, as the reference's checked reader sees the packet's zeroed padding.  A row's reader runs to the
 *     end of the packet, not of its coding unit (init_get_bits is given the rest of the packet), so rows of the first field may read the
 *     second field's bytes; truncated and damaged rows decode exactly as the reference decodes them.
 *  3. Malformed input decodes as the reference decodes it: (2 level + 1) qscale weight wraps in 32 bits, each coefficient is truncated to
 *     int16, last_dc accumulates unclipped and is stored truncated, the "ac tex damaged" break (a run past coefficient 63) leaves the bit
 *     position where it is and the next block starts there, and mbaff (10-bit qscale and the interlaced_mb flag) is honoured on every CID.
 * The codebooks are not restated: `cids` / `n_cids` is the caller's CID table (the decoder's ff_dnxhd_cid_table), searched for each header's
 * CID as ff_dnxhd_get_cid_table does.  The VLC tables are built from the entry and cached by its address, rebuilt when its checksum changes.
 * Refusals beyond the reference's own (each -1 with a message):
 *  - CID 0: a fresh context takes it for its cached CID and never sets cid_table (the reference dereferences NULL);
 *  - a CID entry whose AC, DC or run codes are not a complete prefix code (the reference indexes ac_level[-1] or skips -1 bits on a missing
 *    code), have an AC or run code longer than 16 bits or a DC code longer than 7 (the reference's one-level DC lookup cannot reach it);
 *  - a CID entry whose AC codes need more than 24, or whose run codes need more than 32, second-level tables of the library's lookup (a
 *    9-bit first level, 7-bit second levels; the tables are sized for shared memory, and the entries of ff_dnxhd_cid_table need at most
 *    14 and 24), although the reference's init_vlc accepts such a code;
 *  - a header bit depth other than the entry's bit_depth (init_vlc then reads bit_depth + 4 DC codes from an array of another length);
 *  - an interlaced packet whose second coding unit is not itself an interlaced field header with the first unit's CID, bit depth, chroma
 *    format and size (the reference would reallocate the frame there, or rewrite the first field with a stale cur_field);
 *  - a scan index within 0x280 of 2^32 (the reference's bound check wraps and it reads outside the packet). */
#define FF_DNXHD_PIX_FMT_YUV422P   4     /* AV_PIX_FMT_YUV422P */
#define FF_DNXHD_PIX_FMT_YUV422P10 66    /* AV_PIX_FMT_YUV422P10 (little-endian) */
#define FF_DNXHD_PIX_FMT_YUV444P10 70    /* AV_PIX_FMT_YUV444P10 (little-endian) */
/* What the decoder sets up for a packet before get_buffer. */
typedef struct FFDnxhdFrameInfo {
    int cid;
    int width, height;           /* width: the entry's (the decoder overrides the header's); height: doubled for fields, as dnxhd_decode_header
                                  * does when the header's height matches mb_height */
    int pix_fmt;                 /* FF_DNXHD_PIX_FMT_* */
    int interlaced_frame, top_field_first;
    int sar_num, sar_den;        /* av_reduce(header width, entry width, 255) when they differ, else 0 / 1 (a fresh context's) */
    int lines;                   /* lines each plane must hold: (mb_height * 16) << interlaced_frame, the larger field's mb_height; the decoder
                                  * writes whole macroblocks (1088 lines for 1080p) */
} FFDnxhdFrameInfo;
/* dnxhd_decode_header's checks for the packet (both coding units of an interlaced one) and ff_set_dimensions's, on the host; nothing is
 * launched.  Returns 0, the AVERROR the reference returns (AVERROR_INVALIDDATA, AVERROR(ENOSYS) for an unknown CID, AVERROR(EINVAL) for a
 * size av_image_check_size refuses), or -1 with a message for a refusal listed above.  A decoder calls it in place of dnxhd_decode_header,
 * then ff_set_dimensions and get_buffer as now. */
int ff_dnxhd_probe_cuda(const uint8_t *pkt /* host */, int size, const FFDnxhdCidEntry *cids, int n_cids, FFDnxhdFrameInfo *info);
/* One packet for ff_dnxhd_decode_frames_cuda. */
typedef struct FFDnxhdDecodeWork {
    const uint8_t *pkt_host;     /* the packet on the host, for its headers */
    const uint8_t *pkt;          /* the same bytes on the device */
    int size;
    uint8_t *data[3];            /* device planes: 8-bit samples, or 16-bit samples at 10 bit (even addresses) */
    int linesize[3];             /* bytes between lines: positive, even at 10 bit, at least the plane's width in bytes; U and V equal (the
                                  * reference steps through V with U's linesize) */
    int lines[3];                /* lines each plane holds: at least FFDnxhdFrameInfo.lines */
    int gray;                    /* AV_CODEC_FLAG_GRAY: the chroma planes are left untouched */
} FFDnxhdDecodeWork;
/* Bytes of device workspace ff_dnxhd_decode_frames_cuda needs for these packets (host only, nothing launched); 0 for a batch with a packet
 * or plane the decode call refuses. */
size_t ff_dnxhd_decode_workspace_cuda(const FFDnxhdDecodeWork *works /* host array */, int n, const FFDnxhdCidEntry *cids, int n_cids);
/* dnxhd_decode_frame for n packets on `stream`, without synchronising: every sample the reference decoder writes is written with its value,
 * and nothing else.  Every packet is checked (ff_dnxhd_probe_cuda's checks, then the planes) before anything is launched; -1 with a message
 * for a packet the probe does not accept, NULL or odd planes, linesizes that are not positive, even at 10 bit and as wide as the plane, U and V
 * linesizes that differ, planes with fewer lines than the frame needs, a NULL device packet, and a workspace smaller than
 * ff_dnxhd_decode_workspace_cuda returns. */
int ff_dnxhd_decode_frames_cuda(const FFDnxhdDecodeWork *works /* host array */, int n, const FFDnxhdCidEntry *cids, int n_cids, void *workspace,
                                size_t workspace_bytes, void *stream);

/* ff_xvid_idct / xvid_idct_put / xvid_idct_add (libavcodec/xvididct.c:272-331) over n blocks -- the IDCT ff_xvid_idct_init() installs for
 * MPEG-4 streams written by Xvid and for idct_algo FF_IDCT_XVID.  Arguments, addressing, mode 0 / 1 / 2 and `clear` exactly as
 * ff_simple_idct_batch_cuda; mode 2 leaves the transform result in the blocks.  Blocks at any 2-byte alignment and destinations at any
 * byte alignment are accepted: a batch whose blocks are not 16-byte aligned, or whose frame or stride is not a multiple of 8, runs a
 * thread-per-block kernel instead of the staged one (with dst_off, the offsets must then keep 8-byte alignment as well). */
int ff_xvid_idct_batch_cuda(int mode, int16_t *blocks, uint8_t *frame, const uint32_t *dst_off, ptrdiff_t stride,
                            size_t n, int tiles_per_row, int clear, void *stream);

/* ff_faanidct / ff_faanidct_put / ff_faanidct_add (libavcodec/faanidct.c:113-159) over n blocks -- the IDCT of idct_algo FF_IDCT_FAAN.
 * Arguments, addressing, modes, `clear` and alignment rules exactly as ff_xvid_idct_batch_cuda; put / add leave the coefficients untouched,
 * mode 2 leaves the result (int16-truncated) in the blocks.  Bit-exact to the C code built without FMA: float passes whose products with
 * the AAN constants are evaluated in double and rounded to float once per assignment (DESIGN.md section 5). */
int ff_faanidct_batch_cuda(int mode, int16_t *blocks, uint8_t *frame, const uint32_t *dst_off, ptrdiff_t stride,
                           size_t n, int tiles_per_row, int clear, void *stream);

/* BlockDSPContext.clear_block / clear_blocks over n_blocks * 64 coefficients (blockdsp.c:29-37) and
 * fill_block_tab[w16 ? 0 : 1] over n records (blockdsp.c:39-58). */
int ff_clear_blocks_batch_cuda(int16_t *blocks, size_t n_blocks, void *stream);
int ff_fill_blocks_batch_cuda(uint8_t *frame, const uint32_t *dst_off, const uint8_t *value, ptrdiff_t stride,
                              int h, int w16, size_t n, void *stream);

/* Same op with HOST buffers: uploads `blocks` (and `frame` for mode 1), runs the batch in chunks that
 * overlap H2D / kernel / D2H on three streams, downloads frame (or blocks for mode 2) and synchronises.
 * This is the end-to-end call a caller without device-resident data makes.  frame_bytes = size of the
 * host frame buffer that the offsets address. */
int ff_simple_idct_batch_host_cuda(int mode, int16_t *blocks, uint8_t *frame, size_t frame_bytes,
                                   const uint32_t *dst_off, ptrdiff_t stride, size_t n, int tiles_per_row);

/* ---- H.264 (8 bit, 4:2:0, frame macroblocks) ------------------------------------------------------------
 * The reference calls these slots once per block / partition / edge from its macroblock loop
 * (libavcodec/h264_mb_template.c:40-, h264_mb.c:204-320, h264_loopfilter.c:238-418).  The batched entry points take
 * the same information as arrays of per-macroblock records plus the picture planes, all DEVICE memory. */

/* Inverse quantisation, alone and fused in front of the simple IDCT: MpegEncContext.dct_unquantize_{mpeg1,mpeg2,h263}_
 * {intra,inter} (libavcodec/mpegvideo.c:51-270) as used by put_dct() / add_dequant_dct() (mpegvideo.c:1401-1427).
 *   kind 0 mpeg1_intra  1 mpeg1_inter  2 mpeg2_intra  3 mpeg2_intra_bitexact (mismatch control, what
 *        AV_CODEC_FLAG_BITEXACT installs, mpegvideo.c:281-282)  4 mpeg2_inter  5 h263_intra  6 h263_inter
 * One record per block carries what the C functions read from the MpegEncContext for that block.
 * ff_mpeg_dequant_batch_cuda rewrites the blocks in place (inter kinds leave a block with last_index < 0 untouched,
 * like add_dequant_dct); ff_mpeg_dequant_idct_batch_cuda = dequantise + ff_simple_idct_put (intra kinds) or
 * ff_simple_idct_add (inter kinds; blocks with last_index < 0 are skipped) in one kernel, destinations addressed like
 * ff_simple_idct_batch_cuda.  `tables` is a host struct, everything else device memory.
 * Domain: any int16 level, qscale <= 112, matrix entries <= 255 (so |level| * qscale * matrix stays below 2^31, as it
 * does for every conforming stream); outside it the C code's 32-bit wrap-around is not reproduced. */
typedef struct FFMpegDequantBlock {
    uint8_t qscale;
    int8_t  last_index;    /* s->block_last_index[n] */
    uint8_t dc_scale;      /* n < 4 ? s->y_dc_scale : s->c_dc_scale (intra kinds) */
    uint8_t flags;         /* bit 0: s->ac_pred (h263_intra) */
} FFMpegDequantBlock;
typedef struct FFMpegDequantTables {
    uint16_t intra_matrix[64], inter_matrix[64];   /* s->intra_matrix / s->inter_matrix, raster order */
    uint8_t  permutated[64];                       /* s->intra_scantable.permutated (idctdsp.c:28-47) */
    uint8_t  raster_end[64];                       /* s->inter_scantable.raster_end */
    int      alternate_scan, h263_aic;
} FFMpegDequantTables;
int ff_mpeg_dequant_batch_cuda(int kind, const FFMpegDequantTables *tables, const FFMpegDequantBlock *recs, int16_t *blocks,
                               size_t n, void *stream);
int ff_mpeg_dequant_idct_batch_cuda(int kind, const FFMpegDequantTables *tables, const FFMpegDequantBlock *recs, int16_t *blocks,
                                    uint8_t *frame, const uint32_t *dst_off, ptrdiff_t stride, size_t n, int tiles_per_row,
                                    int clear, void *stream);

/* put_dct / add_dequant_dct (mpegvideo.c:1401-1427) with the Xvid IDCT: same arguments, kinds and skipping rules as
 * ff_mpeg_dequant_idct_batch_cuda, the transform of ff_xvid_idct_batch_cuda.  Blocks must be 16-byte aligned, frame and stride multiples
 * of 8 (and dst_off entries too); anything else is refused. */
int ff_mpeg_dequant_xvid_idct_batch_cuda(int kind, const FFMpegDequantTables *tables, const FFMpegDequantBlock *recs, int16_t *blocks,
                                         uint8_t *frame, const uint32_t *dst_off, ptrdiff_t stride, size_t n, int tiles_per_row,
                                         int clear, void *stream);

/* Residual: H264DSPContext.h264_idct_add16 / _add16intra / idct8_add4 (+ h264_idct_add8 for chroma)
 * (libavcodec/h264idct_template.c:174-214).  Record i consumes coeffs + i * coeff_stride (int16; block k of the MB at
 * + 16 * k, luma k = 0..15, cb 16..19, cr 32..35 -- the reference's sl->mb layout) and nnzc + i * 120
 * (non_zero_count_cache, scan8 addressing, libavcodec/h264dec.h:631-645).  Block offsets are the frame-MB defaults
 * (libavcodec/h264_slice.c:486-493).  Consumed coefficients are zeroed exactly as the C functions zero them. */
typedef struct FFH264ResidualMB {
    uint32_t luma_off;     /* byte offset of the MB origin in the luma plane */
    uint32_t chroma_off;   /* byte offset of the MB origin in the cb / cr planes */
    uint8_t  luma_mode;    /* 0 idct_add16, 1 idct_add16intra, 2 idct8_add4, 3 no luma residual */
    uint8_t  chroma;       /* != 0: run h264_idct_add8 on cb and cr */
    uint8_t  pad[2];
} FFH264ResidualMB;
int ff_h264_idct_add_mb_batch_cuda(const FFH264ResidualMB *mbs, size_t n, int16_t *coeffs, size_t coeff_stride,
                                   const uint8_t *nnzc, uint8_t *luma, uint8_t *cb, uint8_t *cr, int linesize,
                                   int uvlinesize, void *stream);

/* DC transforms + dequantisation, the step hl_decode_mb() runs before the residual of a macroblock:
 * H264DSPContext.h264_luma_dc_dequant_idct (intra 16x16; libavcodec/h264_mb.c:714-719, h264idct_template.c:242-275) from
 * the macroblock's 16 luma DC levels (sl->mb_luma_dc, luma_dc + 16 * i) into the DC positions of its coefficient arena, and
 * h264_chroma_dc_dequant_idct (h264_mb_template.c:182-189, h264idct_template.c:304-324) in place on cb (coeffs + 256) and
 * cr (+ 512).  A qmul of 0 skips that transform (the C code's non_zero_count_cache[...DC_BLOCK_INDEX] test).  Run it on the
 * stream ahead of ff_h264_idct_add_mb_batch_cuda / ff_h264_intra_mb_batch_cuda. */
typedef struct FFH264DCRecord {
    uint32_t luma_qmul;        /* pps->dequant4_coeff[0][qscale][0], 0 = no luma DC block */
    uint32_t chroma_qmul[2];   /* pps->dequant4_coeff[1 + (intra ? 0 : 3)][chroma_qp[0]][0], [2 + ...][chroma_qp[1]][0]; 0 = none */
} FFH264DCRecord;
int ff_h264_dc_dequant_batch_cuda(const FFH264DCRecord *recs, size_t n, int16_t *coeffs, size_t coeff_stride, const int16_t *luma_dc,
                                  void *stream);
/* 8-bit 4:2:2 pictures: the chroma transform is h264_chroma422_dc_dequant_idct (the 2 x 4 DC block, h264idct_template.c:271-306, installed for
 * chroma_format_idc 2 at h264dsp.c:87-90); luma as above */
int ff_h264_dc_dequant_batch_422_cuda(const FFH264DCRecord *recs, size_t n, int16_t *coeffs, size_t coeff_stride, const int16_t *luma_dc,
                                      void *stream);

/* Intra reconstruction: for every intra macroblock of a picture, H264PredContext prediction interleaved with the
 * residual exactly as hl_decode_mb() orders them (libavcodec/h264_mb.c:607-731 hl_decode_mb_predict_luma,
 * h264_mb_template.c:158-197 chroma): intra 4x4 -> per block pred4x4 then idct_add / idct_dc_add; intra 8x8 -> pred8x8l
 * then idct8_add / idct8_dc_add; intra 16x16 -> pred16x16 then h264_idct_add16intra; chroma pred8x8 on cb and cr then
 * h264_idct_add8.  One record per macroblock of the picture in raster order (kind 0 = not intra: its pixels, written by
 * the motion-compensation / residual passes, are only read as neighbours).  Coefficients / nnzc as for
 * ff_h264_idct_add_mb_batch_cuda (DC transforms already applied); consumed coefficients are zeroed like the C code.
 * Rows run as a wavefront two macroblocks behind the row above; progress = mb_h * n_pictures uint32 of scratch.
 * Pictures of a batch are stacked vertically (no prediction across a picture boundary; the records say what is
 * available: the kernel follows topleft / topright_samples_available, not the picture geometry, so slices and
 * constrained_intra_pred are expressed by the masks).  Not covered: transform bypass (the lossless *_add predictors exist
 * as table slots only), MBAFF.
 * Requirements (anything else returns -1 before any work is queued): no NULL pointer; mbs, nnzc and coeffs 4-byte
 * aligned, coeff_stride even and >= 768 (each intra macroblock fetches and writes back the whole 768-element row, blocks
 * 36..47 included, so a shorter stride would overlap the next macroblock's coefficients); luma / cb / cr, linesize and
 * uvlinesize 4-byte aligned.  ff_h264_flush_pictures_cuda checks the same before its first stage when `intra` is set. */
typedef struct FFH264IntraMB {
    uint8_t  kind;             /* 0 not intra, 1 intra 4x4, 2 intra 4x4 with the 8x8 transform (pred8x8l), 3 intra 16x16 */
    uint8_t  mode16;           /* sl->intra16x16_pred_mode (kind 3) */
    uint8_t  chroma_mode;      /* sl->chroma_pred_mode */
    uint8_t  chroma_residual;  /* != 0: h264_idct_add8 after the chroma prediction (cbp & 0x30) */
    uint8_t  mode4[16];        /* sl->intra4x4_pred_mode_cache[scan8[i]]; kind 2 reads entries 0, 4, 8, 12 */
    uint16_t topleft_samples_available, topright_samples_available;   /* h264_mvpred.h:468-508 */
} FFH264IntraMB;
int ff_h264_intra_mb_batch_cuda(const FFH264IntraMB *mbs, int mb_w, int mb_h, int n_pictures, int16_t *coeffs,
                                size_t coeff_stride, const uint8_t *nnzc, uint8_t *luma, uint8_t *cb, uint8_t *cr,
                                int linesize, int uvlinesize, uint32_t *progress, void *stream);

/* Motion compensation: H264QpelContext put/avg tabs + H264ChromaContext put/avg tabs driven like mc_dir_part()
 * (libavcodec/h264_mb.c:204-320): one record = one luma partition and its two chroma partitions.  (x, y) is the
 * partition's luma position, (mvx, mvy) the quarter-pel vector; luma_xy = (mvx & 3) + 4 * (mvy & 3), chroma phase
 * (mvx & 7, mvy & 7).  Reference samples outside the picture are edge-replicated by clamped addressing, which is what
 * emulated_edge_mc (libavcodec/videodsp_template.c:27-94) / the decoder's padded edges provide.
 * All `put` records run before all `avg` records (list 0 then list 1, h264_mb.c:322-366); records of the same kind
 * must address disjoint destination pixels.  A batch of independent pictures is expressed by stacking them vertically
 * (destination and reference planes alike): pic_h is the height of ONE picture and a record with y in
 * [k * pic_h, (k + 1) * pic_h) is clamped to picture k of its reference. */
typedef struct FFH264MCRecord {
    int16_t x, y;          /* luma position of the partition */
    int16_t mvx, mvy;      /* quarter-pel motion vector */
    uint8_t w, h;          /* luma partition size: 16, 8 or 4 each */
    uint8_t avg;           /* 0 put, 1 avg (second prediction direction) */
    uint8_t ref;           /* index into refs[] */
} FFH264MCRecord;
typedef struct FFH264RefPlanes { const uint8_t *y, *cb, *cr; } FFH264RefPlanes;
int ff_h264_mc_batch_cuda(const FFH264MCRecord *recs, size_t n, const FFH264RefPlanes *refs, uint8_t *dst_y, uint8_t *dst_cb,
                          uint8_t *dst_cr, int linesize, int uvlinesize, int pic_w, int pic_h, void *stream);

/* Weighted prediction: H264DSPContext.weight_h264_pixels_tab / biweight_h264_pixels_tab
 * (libavcodec/h264dsp_template.c:30-98) over n rectangles of one plane. */
typedef struct FFH264WeightRecord {
    uint32_t off;          /* byte offset of the block in the plane (dst; src uses the same offset in `src`) */
    uint8_t  w, h;         /* width 16 / 8 / 4 / 2, height */
    uint8_t  log2_denom, pad;
    int16_t  weight, weight_src;   /* weight (uni) or weightd / weights (bi) */
    int16_t  offset, pad2;
} FFH264WeightRecord;
int ff_h264_weight_batch_cuda(const FFH264WeightRecord *recs, size_t n, uint8_t *plane, const uint8_t *src /* NULL = uni */,
                              int stride, void *stream);

/* Deblocking: the 12 loop-filter slots of H264DSPContext (libavcodec/h264dsp_template.c:104-328) applied in the
 * reference's order (macroblocks in raster order; inside one: vertical edges 0..3 then horizontal edges 0..3,
 * libavcodec/h264_loopfilter.c:397-415) to a whole picture.  One record per macroblock, raster order, carrying what
 * filter_mb_edge{v,h,cv,ch} (h264_loopfilter.c:104-236) pass to the slots.  Macroblock rows run as a wavefront that
 * stays two macroblocks behind the row above, so the result is bit-identical to the serial order.
 * dir 0 = vertical edges (h264_h_loop_filter_*), dir 1 = horizontal edges (h264_v_loop_filter_*).
 * An edge with alpha == 0 or beta == 0 is skipped (h264_loopfilter.c:112). */
typedef struct FFH264DeblockMB {
    uint8_t alpha[2][4], beta[2][4];
    int8_t  tc0[2][4][4];          /* per 4-line group, < 0 = group not filtered; ignored on intra edges */
    uint8_t intra[2];              /* bit e set: edge e uses the *_intra (bS = 4) filter */
    uint8_t calpha[2][2][2], cbeta[2][2][2];   /* [plane cb/cr][dir][chroma edge 0/1 = luma edge 0/2] */
    int8_t  ctc0[2][2][2][4];      /* as passed to the chroma slots (already +1), <= 0 = group not filtered */
    uint8_t cintra[2][2];          /* [plane][dir], bit e */
    uint8_t pad[2];
} FFH264DeblockMB;
int ff_h264_deblock_picture_cuda(const FFH264DeblockMB *mbs, int mb_w, int mb_h, uint8_t *luma, uint8_t *cb, uint8_t *cr,
                                 int linesize, int uvlinesize, uint32_t *progress /* 2 * mb_h uint32, scratch */, void *stream);
/* n_pictures independent pictures in one launch: their planes are stacked vertically (picture k starts at luma row
 * k * 16 * mb_h / chroma row k * 8 * mb_h of the same allocations), records likewise (k * mb_w * mb_h);
 * progress holds 2 * mb_h * n_pictures words. */
int ff_h264_deblock_batch_cuda(const FFH264DeblockMB *mbs, int mb_w, int mb_h, int n_pictures, uint8_t *luma, uint8_t *cb,
                               uint8_t *cr, int linesize, int uvlinesize, uint32_t *progress, void *stream);

/* The same three stages for 9 / 10-bit pictures (the BIT_DEPTH > 8 instances, libavcodec/bit_depth_template.c:49-67: uint16 samples,
 * int32 coefficients -- coeffs / coeff_stride count int32 elements, 16 per block like the 8-bit layout; every pitch and every record
 * offset stays in BYTES) and, for the residual and the motion compensation, chroma_format_idc 2 (4:2:2: 8 x 16 chroma macroblocks,
 * h264_idct_add8_422 h264idct_template.c:216-236, chroma vectors at full vertical resolution h264_mb.c:287-316).  Records, order rules
 * and picture stacking are those of the 8-bit calls above; alpha / beta / tc0 in FFH264DeblockMB are the 8-bit-scale table values the
 * decisions produce (the filters scale them by 2^(bit_depth - 8) like h264dsp_template.c:110-113,240).  Field pictures of a frame are
 * pictures in their own right here: pass the field's first row and twice the frame's pitch.  MBAFF frames are not covered.
 * The residual and the motion compensation also take bit_depth 8 with chroma_format_idc 2 (8-bit 4:2:2 pictures: uint8 samples, and `coeffs`
 * then points at int16 coefficients, coeff_stride counting int16); 8-bit 4:2:0 stays with the calls without _hbd, which refuse nothing here. */
int ff_h264_idct_add_mb_batch_hbd_cuda(int bit_depth, int chroma_format_idc, const FFH264ResidualMB *mbs, size_t n, int32_t *coeffs,
                                       size_t coeff_stride, const uint8_t *nnzc, uint8_t *luma, uint8_t *cb, uint8_t *cr, int linesize,
                                       int uvlinesize, void *stream);
int ff_h264_mc_batch_hbd_cuda(int bit_depth, int chroma_format_idc, const FFH264MCRecord *recs, size_t n, const FFH264RefPlanes *refs,
                              uint8_t *dst_y, uint8_t *dst_cb, uint8_t *dst_cr, int linesize, int uvlinesize, int pic_w, int pic_h,
                              void *stream);
int ff_h264_deblock_batch_hbd_cuda(int bit_depth, const FFH264DeblockMB *mbs, int mb_w, int mb_h, int n_pictures, uint8_t *luma,
                                   uint8_t *cb, uint8_t *cr, int linesize, int uvlinesize, void *stream);
/* weighted prediction and the DC transforms for the same pictures: weight_h264_pixels / biweight_h264_pixels at 9 / 10 bit (the record's offset is
 * in 8-bit units and scaled by 2^(bit_depth - 8) like h264dsp_template.c:39,70; `off` and `stride` in bytes) and h264_luma_dc_dequant_idct /
 * h264_chroma_dc_dequant_idct / h264_chroma422_dc_dequant_idct on int32 coefficients (h264idct_template.c:242-324; luma_dc = 16 int32 per macroblock) */
int ff_h264_weight_batch_hbd_cuda(int bit_depth, const FFH264WeightRecord *recs, size_t n, uint8_t *plane, const uint8_t *src /* NULL = uni */,
                                  int stride, void *stream);
int ff_h264_dc_dequant_batch_hbd_cuda(int chroma_format_idc, const FFH264DCRecord *recs, size_t n, int32_t *coeffs, size_t coeff_stride,
                                      const int32_t *luma_dc, void *stream);
/* intra reconstruction at 9 / 10 bit (4:2:0): ff_h264_intra_mb_batch_cuda's records and order, uint16 samples, int32 coefficients; no scratch
 * argument (the wavefront's progress lives in shared memory, one CTA per picture) */
int ff_h264_intra_mb_batch_hbd_cuda(int bit_depth, const FFH264IntraMB *mbs, int mb_w, int mb_h, int n_pictures, int32_t *coeffs,
                                    size_t coeff_stride, const uint8_t *nnzc, uint8_t *luma, uint8_t *cb, uint8_t *cr, int linesize,
                                    int uvlinesize, void *stream);
/* intra reconstruction of 4:2:2 pictures, bit_depth 8 / 9 / 10: the chroma macroblock is 8 x 16 -- pred8x8[] holds the 8 x 16 predictors
 * (h264pred.c:477-563, h264pred_template.c:502-838) and the chroma residual is h264_idct_add8_422 (h264idct_template.c:216-236: blocks 20..23 /
 * 36..39 of the arena, counted at scan8[i + 4]).  coeffs: int16 at 8 bit, int32 at 9 / 10 (coeff_stride in elements of that type). */
int ff_h264_intra_mb_batch_422_cuda(int bit_depth, const FFH264IntraMB *mbs, int mb_w, int mb_h, int n_pictures, void *coeffs,
                                    size_t coeff_stride, const uint8_t *nnzc, uint8_t *luma, uint8_t *cb, uint8_t *cr, int linesize,
                                    int uvlinesize, void *stream);
/* chroma_format_idc 2, bit depth 8 / 9 / 10: the 8 x 16 chroma macroblock has two vertical edges of sixteen lines (the 104-byte record's
 * calpha / cbeta / ctc0 / cintra [plane][0][edge]: h264_h_loop_filter_chroma422, a tc0 entry per four lines) and FOUR horizontal edges, one per
 * luma edge at chroma rows 0, 4, 8, 12 (h264_loopfilter.c:633,693-700: also inside 8x8-transform macroblocks), carried by a second record per
 * macroblock; luma is filtered from the 104-byte record as always ([plane][1][..] of its chroma fields is not read). */
typedef struct FFH264DeblockChroma422 {
    uint8_t alpha[2][4], beta[2][4];   /* [plane cb / cr][edge] */
    int8_t  tc0[2][4][4];              /* as passed to h264_v_loop_filter_chroma (already + 1), <= 0 = group not filtered */
    uint8_t intra[2];                  /* bit e: edge e uses the intra (bS 4) filter */
    uint8_t pad[2];
} FFH264DeblockChroma422;
int ff_h264_deblock_batch_422_cuda(int bit_depth, const FFH264DeblockMB *mbs, const FFH264DeblockChroma422 *chroma422, int mb_w, int mb_h,
                                   int n_pictures, uint8_t *luma, uint8_t *cb, uint8_t *cr, int linesize, int uvlinesize, void *stream);

/* Deblocking DECISIONS (SURVEY 8f rank 1): what loop_filter() -> fill_filter_caches() -> ff_h264_filter_mb()
 * (libavcodec/h264_slice.c:1972-2262, libavcodec/h264_loopfilter.c:438-846) decide for every macroblock of a
 * progressive picture -- boundary strengths, averaged qp, alpha / beta / tc0 per edge -- computed on the
 * device from the decoder's side-information arrays, written as the FFH264DeblockMB records the deblocking kernels
 * above consume.  ff_h264_deblock_params_cuda decides for 8-bit pictures; ff_h264_deblock_params_hbd_cuda takes the bit depth
 * (8, 9 or 10; 8 gives exactly what ff_h264_deblock_params_cuda gives, any other is refused and `out` left untouched).  At 9 / 10 bit
 * qscale_table and chroma_qp_table are the decoder's, in the QP' scale (0..51 + 6 * (bit_depth - 8); I_PCM macroblocks hold 0), and
 * qp_thresh carries its + 6 * (bit_depth - 8) term; the records still hold the 8-bit-scale alpha / beta / tc0 of the reference's tables
 * (h264_loopfilter.c:256-258,726-728), which ff_h264_deblock_batch_hbd_cuda / ff_h264_deblock_batch_422_cuda scale.  All pointers are DEVICE pointers to copies of the decoder's own arrays, in the decoder's layouts:
 *   mb_type, qscale_table, cbp_table, slice_table: [n_pictures * mb_h][mb_w + 1] (mb_stride = mb_w + 1, the extra
 *       column is the decoder's padding and is never read)          H264Picture.mb_type / qscale_table, H264Context
 *   non_zero_count: [..][48] per macroblock                          H264Context.non_zero_count
 *   motion_val[list]: [4 * n_pictures * mb_h][4 * mb_w][2] int16     H264Picture.motion_val, b_stride = 4 * mb_w
 *   ref_index[list]: [..][4] per macroblock (one per 8x8)            H264Picture.ref_index
 *   slices[slice_num]: the slice-header values the filter uses and the slice's ref2frm table (h264dec.h:186,538;
 *       ref2frm[list][2 + ref_index] = identity of the referenced frame, entries 0/1 = -1); at most 32 slice numbers
 *   chroma_qp_table: PPS.chroma_qp_table[2][64] (h264_ps.h:124)
 * Pictures of a batch are stacked row-wise; no edge is filtered across a picture boundary.
 * Field pictures (PAFF) are covered through field_picture, 4:2:2 through chroma422; not covered: MBAFF frames, 4:4:4 (the records
 * themselves are bit-depth agnostic: ff_h264_deblock_batch_hbd_cuda takes them for 9 / 10-bit pictures). */
typedef struct FFH264DeblockSlice {
    int32_t alpha_c0_offset, beta_offset;   /* sl->slice_alpha_c0_offset, sl->slice_beta_offset */
    int32_t deblocking_filter;              /* 0 off, 1 every edge, 2 not across slice boundaries */
    int32_t list_count;                     /* 1 (P) or 2 (B) */
    int32_t qp_thresh;                      /* sl->qp_thresh, h264_slice.c:1815-1818 */
    int32_t ref2frm[2][64];
} FFH264DeblockSlice;
typedef struct FFH264DeblockInfo {
    int mb_w, mb_h, n_pictures;
    const uint32_t *mb_type;
    const int8_t   *qscale_table;
    const uint8_t  *non_zero_count;
    const uint16_t *cbp_table, *slice_table;
    const int16_t  *motion_val[2];
    const int8_t   *ref_index[2];
    const FFH264DeblockSlice *slices;
    int n_slices;
    const uint8_t  *chroma_qp_table;
    int cabac, transform_8x8_mode;          /* PPS.cabac, PPS.transform_8x8_mode */
    int field_picture;                      /* h->picture_structure != PICT_FRAME: the pictures are fields (every mb_type carries
                                               MB_TYPE_INTERLACED): vertical vector limit 2, bS 3 on horizontal intra macroblock edges
                                               (h264_loopfilter.c:551-557,723) */
    FFH264DeblockChroma422 *chroma422;      /* device pointer, NULL for 4:2:0; else chroma_format_idc 2: the horizontal chroma edges of
                                               macroblock m are written to chroma422[m] instead of the 104-byte record's [plane][1][..] */
} FFH264DeblockInfo;
int ff_h264_deblock_params_cuda(const FFH264DeblockInfo *info /* host struct */, FFH264DeblockMB *out, void *stream);
int ff_h264_deblock_params_hbd_cuda(int bit_depth, const FFH264DeblockInfo *info /* host struct */, FFH264DeblockMB *out, void *stream);

/* The flush point of a decoder back-end (SURVEY 8f rank 1): the CPU parses and entropy-decodes, RECORDS the work of a batch of
 * pictures (or of the slices decoded so far) in the arrays below, and flushes it with one call.  The stages run on `stream` in
 * the order hl_decode_mb() (libavcodec/h264_mb_template.c:40-260: inter prediction, weighted prediction, DC transforms,
 * residual; intra prediction interleaved with its residual) and loop_filter() (libavcodec/h264_slice.c:1972-2066) impose; the
 * call returns without synchronising.  Every array is a DEVICE pointer (deblock_info is a host struct of device pointers), a
 * NULL array / zero count skips its stage.  Per-macroblock arrays (dc, residual, intra, deblock_records, the coefficient arena
 * coeffs + i * coeff_stride, nnzc + i * 120) have one entry per macroblock of the batch in raster order, pictures stacked:
 * a macroblock that takes no part in a stage says so in its record (residual luma_mode 3 / chroma 0 for intra and skipped
 * macroblocks, intra kind 0 for inter ones, dc qmul 0).  Planes: n_pictures pictures stacked vertically, 16 * mb_h luma rows
 * each.  progress: 2 * mb_h * n_pictures uint32 of scratch. */
typedef struct FFH264PictureWork {
    int mb_w, mb_h, n_pictures;
    uint8_t *luma, *cb, *cr;                 /* the pictures being reconstructed */
    int linesize, uvlinesize;
    const FFH264MCRecord *mc; size_t n_mc;   /* ff_h264_mc_batch_cuda; pic_w / pic_h = 16 * mb_w / 16 * mb_h */
    const FFH264RefPlanes *refs;
    const FFH264WeightRecord *weight[3]; size_t n_weight[3];   /* per plane: ff_h264_weight_batch_cuda */
    const uint8_t *weight_src[3];            /* bi-weighting: the plane holding the second prediction, else NULL */
    int16_t *coeffs; size_t coeff_stride;    /* coefficient arena, consumed (zeroed) like the C functions do */
    const uint8_t *nnzc;
    const FFH264DCRecord *dc; const int16_t *luma_dc;          /* ff_h264_dc_dequant_batch_cuda */
    const FFH264ResidualMB *residual;        /* ff_h264_idct_add_mb_batch_cuda */
    const FFH264IntraMB *intra;              /* ff_h264_intra_mb_batch_cuda */
    const FFH264DeblockInfo *deblock_info;   /* host struct: decisions are derived on the device into deblock_records */
    FFH264DeblockMB *deblock_records;        /* with deblock_info NULL: records the caller already filled; NULL = no loop filter */
    uint32_t *progress;
    int bit_depth, chroma_format_idc;        /* 0 = 8 / 1.  9 / 10-bit pictures (int32 coeffs / luma_dc behind the same pointers) and 4:2:2 chroma at
                                                8 / 9 / 10 bit run the *_hbd_cuda / *_422_cuda stages in the same order (progress is not used then;
                                                4:2:2 intra macroblocks: ff_h264_intra_mb_batch_422_cuda; decisions from deblock_info:
                                                ff_h264_deblock_params_hbd_cuda at bit_depth, so its side information is in the QP' scale) */
    const FFH264DeblockChroma422 *deblock_chroma422;   /* 4:2:2 with caller-filled deblock_records: their second record array */
} FFH264PictureWork;
int ff_h264_flush_pictures_cuda(const FFH264PictureWork *work /* host struct */, void *stream);

/* ---- MECmpContext, motion search, HpelDSPContext, FDCTDSPContext -----------------------------------------
 * me_cmp: n block pairs (cur + cur_off vs ref + ref_off, common stride, height h) through one metric; out[i] is
 * what the C slot returns.  kind / sidx / dxy select the slot like the reference's tables (libavcodec/me_cmp.h:39-63):
 *   kind 0 pix_abs[sidx][dxy] (sidx 0 = 16 wide, 1 = 8 wide; dxy = x2 + 2*y2 half-pel flag)   me_cmp.c:109-307
 *        1 sad[sidx]   2 sse[sidx] (sidx 2 = 4 wide)   3 hadamard8_diff[sidx]   4 vsad[0]   5 vsse[0]
 *        6 nsse[sidx] (weight 8: the NULL-context default, me_cmp.c:331)   7 hadamard8_diff[4 + sidx] (intra)
 *        8 vsad[4 + sidx] (intra)   9 vsse[4 + sidx] (intra)   10 sum_abs_dctelem (cur_off in bytes into int16 blocks)
 *       11 dct_sad[sidx]   12 dct_max[sidx]   13 dct264_sad[sidx]   (me_cmp.c:538-621; for 11 / 12 `dxy` names the
 *          FDCTDSPContext.fdct the encoder context holds: 0 = ff_jpeg_fdct_islow_8, 2 = ff_fdct_ifast, 6 = ff_faandct)
 * These three only dereference the MpegEncContext's DSP tables, so the batch call covers them; their table slots are
 * left to the C code (a slot cannot know which fdct the caller's context selected).  quant_psnr, bit and rd
 * (me_cmp.c:621-782) need the quantiser and VLC length tables of a live encoder: see ff_me_cmp_enc_batch_cuda below. */
typedef struct FFMECmpRecord { uint32_t cur_off, ref_off; } FFMECmpRecord;
int ff_me_cmp_batch_cuda(int kind, int sidx, int dxy, const uint8_t *cur, const uint8_t *ref, ptrdiff_t stride, int h,
                         const FFMECmpRecord *recs, size_t n, int32_t *out, void *stream);

/* quant_psnr / bit / rd (libavcodec/me_cmp.c:621-782: quant_psnr8x8_c, bit8x8_c, rd8x8_c and their 16-wide wrappers :883-885): the three
 * metrics that run the encoder's own quantiser on the difference block -- s->fast_dct_quantize = ff_dct_quantize_c
 * (libavcodec/mpegvideo_enc.c:773-777, :4371-4450: forward DCT, DC division, biased threshold quantiser in scan order) -- then count
 * VLC bits from the codec's run / level length tables (bit, rd) and / or reconstruct through s->dct_unquantize_intra / _inter
 * (libavcodec/mpegvideo.c:51-270) and the simple IDCT (quant_psnr, rd).  FFMECmpEncState = the MpegEncContext fields they read, by value
 * (q_*_matrix = the row of s->q_intra_matrix / s->q_inter_matrix for `qscale`, as ff_convert_matrix() built it, mpegvideo_enc.c:84-160);
 * FFMECmpVlcTables = the codec's static length tables (HOST pointers; [64 * 128] indexed UNI_AC_ENC_INDEX(run, level + 64), the DC table
 * [512] indexed level + 256; may be NULL for quant_psnr, which reads none).  The IDCT is the table's own: FF_IDCT_PERM_NONE
 * (what ff_idctdsp_init_cuda installs), so scantable serves the quantiser and the bit counter alike.
 *   kind 14 quant_psnr (always quantises as an inter block, like the C code)   15 bit   16 rd;   sidx 0 = 16 wide (h 16 or 8), 1 = 8x8
 *   out[i] = the slot's return value; last_index[i] (optional) = s->block_last_index[0] as the C function leaves it.
 * A DC level outside the DC table (|level| > 255: impossible for 8-bit differences with dc_scale >= 1) is clamped to its ends. */
typedef struct FFMECmpEncState {
    int32_t fdct;                  /* s->fdsp.fdct: 0 ff_jpeg_fdct_islow_8, 2 ff_fdct_ifast, 6 ff_faandct */
    int32_t dequant;               /* s->dct_unquantize_intra / _inter (mpegvideo_enc.c:1613-1622): 0 mpeg1, 1 mpeg2, 2 mpeg2 under
                                      AV_CODEC_FLAG_BITEXACT (mismatch control on intra blocks too), 3 h263 */
    int32_t qscale, mb_intra, y_dc_scale, h263_aic;
    int32_t intra_quant_bias, inter_quant_bias, ac_esc_length;
    int32_t q_intra_matrix[64], q_inter_matrix[64];
    uint16_t intra_matrix[64], inter_matrix[64];   /* s->intra_matrix / s->inter_matrix (the inverse quantisers' side) */
    uint8_t scantable[64];                         /* s->intra_scantable.scantable */
} FFMECmpEncState;
typedef struct FFMECmpVlcTables {
    const uint8_t *intra_ac_vlc_length, *intra_ac_vlc_last_length, *inter_ac_vlc_length, *inter_ac_vlc_last_length, *luma_dc_vlc_length;
} FFMECmpVlcTables;
/* device-resident copy of one encoder state (one per (qscale, mb_intra) a batch uses); NULL + avb200_last_error() on failure */
void *ff_me_cmp_enc_state_cuda(const FFMECmpEncState *state, const FFMECmpVlcTables *vlc);
void ff_me_cmp_enc_state_free_cuda(void *enc_state);
int ff_me_cmp_enc_batch_cuda(int kind, int sidx, const void *enc_state, const uint8_t *cur, const uint8_t *ref, ptrdiff_t stride, int h,
                             const FFMECmpRecord *recs, size_t n, int32_t *out, int32_t *last_index, void *stream);

/* ---- the mpegvideo encoders' quantiser (MPEG-1 / MPEG-2, H.263 / MPEG-4 part 2, MJPEG; 8 bit) --------------------------------------------
 * What encode_mb_internal (libavcodec/mpegvideo_enc.c:2263-2303) does to every coded block between the pixel fetch and the VLC pass:
 *   s->dct_quantize: the forward DCT (s->fdsp.fdct), denoise_dct_c when noise reduction is on (:3621-3643), then ff_dct_quantize_c
 *   (:4371-4450) or, with trellis, dct_quantize_trellis_c (:3645-3936); clip_coeffs (:1951-1983) when the quantiser reports overflow;
 *   dct_single_coeff_elimination (:1895-1949) on inter blocks when the block's threshold (luma for blocks 0-3, chroma for the rest) is not 0.
 * FFMpvQuantState = the MpegEncContext fields those functions read that stay fixed over a picture, by value: q_intra_matrix / q_inter_matrix
 * for every qscale as ff_convert_matrix() built them (mpegvideo_enc.c:84-160), scantable = s->intra_scantable.scantable.  The IDCT must not
 * permute (FF_IDCT_PERM_NONE), so levels come back in raster order exactly as the C code leaves s->block[n].  FFMpvQuantRecord = the fields
 * that change per macroblock or block.  The trellis also reads the codec's VLC length tables (FFMECmpVlcTables: the same device cache as the
 * quant_psnr / bit / rd metrics; luma_dc_vlc_length is not read and may be NULL).  Under ff_fdct_ifast the trellis weighs its distortion with
 * ff_inv_aanscales, which the library derives from its definition (round(4096 / (a(u) a(v))), a(0) = 1, a(k) = sqrt(2) cos(k pi / 16)). */
typedef struct FFMpvQuantState {
    int32_t fdct;                                   /* s->fdsp.fdct: 0 ff_jpeg_fdct_islow_8, 2 ff_fdct_ifast, 6 ff_faandct */
    int32_t out_format;                             /* enum OutputFormat (mpegutils.h): 0 FMT_MPEG1, 1 FMT_H261, 2 FMT_H263, 3 FMT_MJPEG */
    int32_t mpeg_quant, h263_aic;
    int32_t intra_quant_bias, inter_quant_bias;     /* QUANT_BIAS_SHIFT units; the trellis ignores them (its own thresholds) */
    int32_t ac_esc_length, min_qcoeff, max_qcoeff;
    int32_t luma_elim_threshold, chroma_elim_threshold;   /* 0 = off, < 0 = the DC too */
    int32_t q_intra_matrix[32][64], q_inter_matrix[32][64];
    uint16_t intra_matrix[64], inter_matrix[64];
    uint8_t scantable[64];                          /* a permutation of 0..63 with scantable[0] == 0 */
    uint8_t pad[8];
} FFMpvQuantState;
typedef struct FFMpvQuantRecord {                   /* one per block */
    uint8_t qscale;                                 /* 1..31 */
    uint8_t intra;                                  /* s->mb_intra */
    uint8_t dc_scale;                               /* s->y_dc_scale for blocks 0-3, s->c_dc_scale for the others (intra, not h263_aic: >= 1) */
    uint8_t chroma;                                 /* block index n >= 4: picks the elimination threshold */
    uint32_t lambda2;                               /* s->lambda2 of the macroblock (trellis) */
} FFMpvQuantRecord;
typedef struct FFMpvNoiseReduction {                /* DEVICE pointers: s->dct_offset [2][64], s->dct_error_sum [2][64], s->dct_count [2] */
    const uint16_t *dct_offset;
    int32_t *dct_error_sum, *dct_count;
} FFMpvNoiseReduction;
/* device-resident copy of a state (one per picture, or per change of matrices); NULL + avb200_last_error() for a bad state: an fdct other
 * than 0, 2 or 6, an out_format outside 0..3, a scantable that is not a permutation starting at 0.  vlc may be NULL when no call uses trellis. */
void *ff_mpv_quant_state_cuda(const FFMpvQuantState *state, const FFMECmpVlcTables *vlc);
void ff_mpv_quant_state_free_cuda(void *quant_state);
/* n blocks, one thread each, on `stream` without synchronising.  Input: s1 == NULL -> blocks[i] already holds what get_pixels /
 * diff_pixels left there; otherwise the kernel fetches block i itself from s1 + off1[i] (minus s2 + off2[i] when s2 != NULL; off2 NULL = the
 * same offsets), as ff_pixblock_fdct_batch_cuda does.  trellis 0 = ff_dct_quantize_c, 1 = dct_quantize_trellis_c.  Output: blocks[i] =
 * the levels after the clip and the elimination (raster order), last_index[i] = s->block_last_index[n] after them, coded_score[i] (optional)
 * = s->coded_score[n] where the trellis writes it (it is left as it was where the C code leaves it).  nr (host struct of device pointers,
 * NULL = off): the dct_offset the blocks are denoised with, and dct_error_sum / dct_count, which are added to (int32 adds: the C result
 * whatever the block order).  A record with qscale outside 1..31 or an intra dc_scale of 0 (without h263_aic) leaves its block, last_index,
 * coded_score and the sums alone: the records are device memory, so unlike the checks below this one is made by the kernel, per block,
 * and the call still returns 0.  Returns 0 (n == 0 too), or -1 with avb200_last_error() set and nothing launched: no state, trellis on a
 * state without VLC tables, blocks not 16-byte aligned, a NULL buffer. */
int ff_mpv_dct_quantize_batch_cuda(const void *quant_state, int trellis, const FFMpvQuantRecord *recs, const uint8_t *s1, const uint8_t *s2,
                                   const uint32_t *off1, const uint32_t *off2, ptrdiff_t stride, int16_t *blocks, size_t n,
                                   int32_t *last_index, int32_t *coded_score, const FFMpvNoiseReduction *nr, void *stream);

/* Exhaustive search (libavcodec/motion_est_template.c:620-655) for every 16x16 macroblock of rows [mb_y0, mb_y1):
 * candidates within +-range (16) clipped so the block stays inside the picture (get_limits, motion_est.c:517-548),
 * score = pix_abs[0][0] (h = 16), penalty_factor 0, strict-< minimum in raster order (mathops.h:133-140).
 * out[3 * (mb_y * (w / 16) + mb_x)] = { mx, my, sad }.  Sharding over GPUs = disjoint row ranges. */
int ff_full_search_cuda(const uint8_t *cur, const uint8_t *ref, int stride, int w, int h, int range, int mb_y0, int mb_y1,
                        int32_t *out, void *stream);

/* HpelDSPContext (libavcodec/hpeldsp.h:45-93): tab 0 put, 1 avg, 2 put_no_rnd, 3 avg_no_rnd; sidx 0..3 = width
 * 16 / 8 / 4 / 2; dxy = x_halfpel + 2 * y_halfpel; h rows.  dst and src share `stride` like the C slots. */
typedef struct FFHpelRecord { uint32_t dst_off, src_off; uint8_t tab, sidx, dxy, h; } FFHpelRecord;
int ff_hpel_batch_cuda(const FFHpelRecord *recs, size_t n, uint8_t *dst, const uint8_t *src, ptrdiff_t stride, void *stream);

/* QpelDSPContext (libavcodec/qpeldsp.h:69-73): MPEG-4 quarter-pel motion compensation, n blocks per launch.
 * kind 0 put_qpel_pixels_tab, 1 put_no_rnd_qpel_pixels_tab, 2 avg_qpel_pixels_tab; sidx 0 = 16x16, 1 = 8x8;
 * mc = x + 4 * y quarter-pel phase (the table index, qpeldsp.c:734-752).  dst and src share `stride` like the C slots;
 * records of one launch must address disjoint destination blocks. */
typedef struct FFQpelRecord { uint32_t dst_off, src_off; uint8_t kind, sidx, mc, pad; } FFQpelRecord;
int ff_mpeg4_qpel_batch_cuda(const FFQpelRecord *recs, size_t n, uint8_t *dst, const uint8_t *src, ptrdiff_t stride, void *stream);

/* ---- mpegvideo motion compensation (MPEG-1 / MPEG-2 4:2:0 / 4:2:2 / 4:4:4, H.263 / MPEG-4 part 2 4:2:0; 8 bit) ---------------------------
 * ff_mpv_motion() (libavcodec/mpegvideo_motion.c:814-968) for every direction of a macroblock, in ff_mpv_reconstruct_mb's order
 * (mpegvideo.c:1548-1578): the forward prediction with put (put_no_rnd when no_rounding is set in a P picture), then the backward one
 * with avg.  One record per inter macroblock, its fields named after the MpegEncContext fields the C function reads.
 *   MPEG-1 / MPEG-2 (out_format 0): 16X16 in frame pictures; FIELD in frame and field pictures; 16X8 in field pictures; DMV in both.
 *     Chroma 4:2:0, 4:2:2 or 4:4:4 (chroma_format 1, 2, 3: mpeg_motion_internal's chroma cases, :307-326).  A vector whose luma block
 *     leaves [0, h_edge_pos) x [0, v_edge_pos) skips that mpeg_motion call, chroma included, exactly like the C code (:333-342).
 *   H.263 / MPEG-4 (out_format 2): 16X16 half- and quarter-sample, 8X8 (4MV) half- and quarter-sample, with the reference's edge
 *     emulation where it emulates (clamped addressing) and direct reads where it reads directly.  In an interlaced MPEG-4 picture
 *     (interlaced set) also FIELD: mpeg_motion_field for each parity (FF_BUG_HPEL_CHROMA's chroma vector when workaround_bugs has it),
 *     or, quarter-sample, qpel_motion with field_based (two 8x8 qpel ops per field).  Their edge emulation works in frame rows, as
 *     emulated_edge_mc does: field row i of parity f reads frame row av_clip(2 * (src_y + i) + f, 0, v_edge_pos - 1).
 * OBMC: a P picture with obmc set (out_format 2, half-sample, obmc_recs given) runs apply_obmc for each record instead, from its
 *   FFMpvOBMCRecord: the four 8x8 luma blocks as put_obmc weighted sums of hpel_motion predictions (put_no_rnd under no_rounding), chroma
 *   through chroma_4mv_motion with the sum of the four own vectors -- also for a 16X16 macroblock.  Its records must be forward-only
 *   (mv_dir & 3 == 1); others count as rejected.  obmc is ignored in B pictures, as in the C code.
 * GMC: an MPEG-4 S-VOP (sprite set: out_format 2, a frame picture, not b_picture, obmc 0, real_sprite_warping_points 1..3 and
 *   sprite_warping_accuracy 0..3) runs, for a 16X16 record with mcsel set, gmc1_motion (real_sprite_warping_points 1) or gmc_motion
 *   (2, 3) (mpegvideo_motion.c:37-190) from the picture's sprite_offset / sprite_delta, with put for every direction the record names;
 *   its mv is not read.  Every other record of an S-VOP (mcsel 0, 8X8 with mcsel ignored, as in the C code) runs as in a P picture.
 *   The sprite fields must be those mpeg4_decode_sprite_trajectory (mpeg4videodec.c:168-385) leaves: the C arithmetic, which the kernel
 *   follows, is only defined where gmc_motion's and ff_gmc_c's intermediates fit int32 (the kernel's affine map is that arithmetic
 *   mod 2^32 all the same).
 * Refused: static sprites and any other sprite picture, OBMC in a quarter-sample, MPEG-1 / 2, obmc_recs-less or interlaced P picture,
 * H.261, WMV2 mspel, field pictures in the H.263 family, chroma_format outside 1..3 or other than 1 in the H.263 family, lowres.  A picture
 * asking for one of them makes the call return -1 with avb200_last_error() set, and nothing is launched.  A record the kernel cannot
 * take (an mv_type outside the family's list -- FIELD counts as outside it in an H.263-family picture without interlaced, 16X8 and DMV
 * always --, mv_dir above 7, a macroblock outside the picture, a direction whose reference planes are NULL) leaves its macroblock
 * untouched and adds one to *rejected (device uint32).
 * Memory: the kernel reads each reference plane only inside rows [0, 16 * mb_height] and columns [0, 16 * mb_width] (chroma
 * [0, (16 >> chroma_y_shift) * mb_height] x [0, (16 >> chroma_x_shift) * mb_width]: 8 x 8 per macroblock in 4:2:0, 8 wide and 16 high in
 * 4:2:2, 16 x 16 in 4:4:4), whatever the records hold: the macroblock-aligned plane plus one row below and one column to the right.  The C code reads that far directly in one case: in a picture narrower (shorter) than 16 samples, FFMAX(h_edge_pos - 16, 0)
 * lets a 16x16 H.263 / MPEG-4 vector at 0 read the reference directly, and its 9-sample chroma block ends one column (row) past the
 * aligned plane.  Elsewhere direct reads may pass h_edge_pos / v_edge_pos but stay inside the aligned plane.  GMC reads less: gmc1_motion
 * reads a 17 x 17 luma and 9 x 9 chroma window, clamped to [0, h_edge_pos) x [0, v_edge_pos) (halved for chroma) wherever the C code
 * emulates the edge and else inside the aligned plane; gmc_motion reads only inside [0, h_edge_pos) x [0, v_edge_pos).  The kernel writes only the
 * destination macroblocks of accepted records.
 * Records of one picture run concurrently: a picture holds at most one record per macroblock (two records for the same mb_x, mb_y race,
 * and the result is undefined).  Pictures of one call run concurrently too, so none may read what another writes: a second field that
 * predicts from its own first field goes into a later call.  Checked by frame base (dest[0], one line less for a bottom field): two
 * pictures of a call writing the same frame, a picture whose frame is another's last[0] / next[0] or its own, and a cur[0] other than
 * that frame are refused. */
typedef struct FFMpvMCRecord {
    uint16_t mb_x, mb_y;          /* s->mb_x; the macroblock row in the picture: s->mb_y >> field_pic */
    uint8_t  mv_dir;              /* s->mv_dir: bit 0 MV_DIR_FORWARD, bit 1 MV_DIR_BACKWARD (bit 2, MV_DIRECT, is ignored) */
    uint8_t  mv_type;             /* s->mv_type: 0 16X16, 1 8X8, 2 16X8, 3 FIELD, 4 DMV */
    uint8_t  field_select[2][2];  /* s->field_select */
    int16_t  mv[2][4][2];         /* s->mv */
    uint8_t  mcsel;               /* s->mcsel when ff_mpv_reconstruct_mb runs (mpeg4videodec.c:1221-1227, :1333-1336); read in S-VOPs only */
    uint8_t  pad;
} FFMpvMCRecord;
/* H.263 overlapped block motion compensation (Annex F; Intel H.263; RV10 micro-version 2): apply_obmc (mpegvideo_motion.c:643-728), which
 * replaces ff_mpv_motion's prediction in a P picture with obmc set.  It reads current_picture.motion_val[0] and mb_type at the moment the
 * decoder reconstructs the macroblock, and the right neighbour's entries there are not always final (preview_obmc, ituh263dec.c:339-400,
 * is skipped after a skipped macroblock and for the last macroblock of a GOB), so the record carries raw copies of what it reads; the
 * kernel makes the substitutions of :674-700 (a neighbour outside the picture or IS_INTRA is replaced by the macroblock's own vectors).
 * With b8_stride = s->b8_stride, mot_xy = 2 * mb_x + 2 * mb_y * b8_stride and xy = mb_x + mb_y * mb_stride: */
typedef struct FFMpvOBMCRecord {
    int16_t mv[4][2];             /* motion_val[0][mot_xy], [mot_xy + 1], [mot_xy + b8_stride], [mot_xy + b8_stride + 1] */
    int16_t top[2][2];            /* motion_val[0][mot_xy - b8_stride], [mot_xy - b8_stride + 1] (read when mb_y > 0) */
    int16_t left[2][2];           /* motion_val[0][mot_xy - 1], [mot_xy - 1 + b8_stride] (read when mb_x > 0) */
    int16_t right[2][2];          /* motion_val[0][mot_xy + 2], [mot_xy + 2 + b8_stride] (read when mb_x + 1 < mb_width) */
    uint32_t mb_type_top, mb_type_left, mb_type_right;  /* mb_type[xy - mb_stride], [xy - 1], [xy + 1] */
} FFMpvOBMCRecord;
typedef struct FFMpvMCPicture {
    uint8_t *dest[3];                   /* s->current_picture.f->data: the bottom field of a field picture starts one line down */
    const uint8_t *cur[3];              /* s->current_picture_ptr->f->data: the frame's own planes (second field P prediction) */
    const uint8_t *last[3], *next[3];   /* s->last_picture.f->data, s->next_picture.f->data (NULL where no record uses them) */
    int linesize, uvlinesize;           /* s->linesize, s->uvlinesize (frame lines) */
    int pic_linesize, pic_uvlinesize;   /* s->current_picture.f->linesize[0] / [1]: the frame's, doubled in a field picture */
    int mb_width, mb_height;            /* s->mb_width, s->mb_height (frame macroblocks) */
    int width, height, h_edge_pos, v_edge_pos;
    int out_format;                     /* s->out_format: 0 FMT_MPEG1 (MPEG-1 / 2), 2 FMT_H263 (H.263, MPEG-4 part 2); 1 (H.261) is refused */
    int picture_structure;              /* 1 top field, 2 bottom field, 3 frame */
    int first_field, b_picture;         /* s->first_field; s->pict_type == AV_PICTURE_TYPE_B */
    int no_rounding, quarter_sample, workaround_bugs;
    int chroma_format;                  /* s->chroma_format: 1 (4:2:0); 2 (4:2:2) or 3 (4:4:4) with out_format 0 only */
    int obmc, sprite, mspel, lowres;    /* s->obmc; s->pict_type == AV_PICTURE_TYPE_S; s->mspel; avctx->lowres: must be 0 */
    const FFMpvMCRecord *recs;          /* device; at most one record per macroblock */
    size_t n_recs;
    const FFMpvOBMCRecord *obmc_recs;   /* device, one per record in the same order, read when obmc is set in a P picture; else NULL */
    /* read when sprite is set: the MpegEncContext fields as mpeg4_decode_sprite_trajectory leaves them */
    int sprite_warping_accuracy, real_sprite_warping_points;
    int sprite_offset[2][2], sprite_delta[2][2];
    int interlaced;                     /* !s->progressive_sequence, read in out_format 2 only: FIELD records of the frame picture are taken */
} FFMpvMCPicture;
/* put_dct / add_dequant_dct (mpegvideo.c:1401-1427) with the FAAN IDCT: same arguments, kinds, skipping rules and alignment rules as
 * ff_mpeg_dequant_xvid_idct_batch_cuda, the transform of ff_faanidct_batch_cuda. */
int ff_mpeg_dequant_faanidct_batch_cuda(int kind, const FFMpegDequantTables *tables, const FFMpegDequantBlock *recs, int16_t *blocks,
                                        uint8_t *frame, const uint32_t *dst_off, ptrdiff_t stride, size_t n, int tiles_per_row,
                                        int clear, void *stream);

int ff_mpv_motion_batch_cuda(const FFMpvMCPicture *pictures /* host array */, int n_pictures, uint32_t *rejected, void *stream);

/* The flush point of an mpegvideo decoder back-end: the decoder parses a batch of pictures, records the motion of every inter macroblock
 * and the coefficient blocks of every coded block, and flushes with one call.  On `stream`, without synchronising: the motion
 * compensation of every picture (ff_mpv_motion_batch_cuda), then the residual batches in the order given, each through one existing entry
 * point -- the simple or the Xvid transform, with no inverse quantiser or one of the seven kinds of ff_mpeg_dequant_idct_batch_cuda:
 *   dequant -1, transform 0: ff_simple_idct_batch_cuda(mode, ...)        dequant k, transform 0: ff_mpeg_dequant_idct_batch_cuda(k, ...)
 *   dequant -1, transform 1: ff_xvid_idct_batch_cuda(mode, ...)          dequant k, transform 1: ff_mpeg_dequant_xvid_idct_batch_cuda(k, ...)
 *   dequant -1, transform 3: ff_faanidct_batch_cuda(mode, ...)           dequant k, transform 3: ff_mpeg_dequant_faanidct_batch_cuda(k, ...)
 * Intra blocks (idct_put / put_dct) and inter blocks (idct_add / add_dct / add_dequant_dct) go in separate batches, and so do frame and
 * field DCT blocks: a field-DCT block of a macroblock at dest has dct_linesize = 2 * linesize and its lower blocks start one line down
 * (mpegvideo.c:1534-1535).  Blocks are addressed through dst_off (byte offsets into `frame`).  Every batch is checked before anything is
 * launched; a refusal returns -1 and leaves every picture as it was.  A batch its entry point refuses later (its alignment rules) stops
 * the flush with -1 after the stages before it were enqueued.  Then, when loop_filter is set, the H.263 deblocking filter of those pictures
 * (ff_h263_loop_filter_batch_cuda), checked with everything else before the first stage is enqueued. */
typedef struct FFMpvResidualBatch {
    int transform;                       /* 0 simple IDCT, 1 Xvid IDCT, 3 FAAN IDCT (2 is not a transform) */
    int dequant;                         /* -1: the blocks are dequantised already; 0..6: the inverse quantiser kind fused in front */
    int mode;                            /* dequant -1: 0 put, 1 add (a fused kind puts for intra kinds, adds for inter kinds) */
    const FFMpegDequantTables *tables;   /* host struct, dequant >= 0 */
    const FFMpegDequantBlock *recs;      /* device, dequant >= 0 */
    int16_t *blocks;                     /* device, n * 64 */
    uint8_t *frame;                      /* device plane the offsets address */
    const uint32_t *dst_off;             /* device, n */
    ptrdiff_t stride;                    /* linesize, or 2 * linesize for field DCT */
    size_t n;
    int clear;
} FFMpvResidualBatch;

/* ---- H.263 deblocking filter (Annex J; H.263+, RV20) over whole pictures ------------------------------------------------------------
 * What ff_h263_loop_filter (libavcodec/h263.c:135-220) does when the decoder runs it for every macroblock in raster order
 * (h263dec.c:250-252,281-283, rv10.c:654-655), for n pictures, on `stream`, without synchronising.  The filter of a macroblock writes only
 * into it and its left / upper neighbours, and no later reconstruction of an H.263 picture reads the picture itself, so running it after
 * the whole picture has been reconstructed gives the same bytes.  Every macroblock of the macroblock-aligned planes is filtered, the area
 * past width / height of a custom-size picture included; nothing outside rows [0, 16 * mb_height) x columns [0, 16 * mb_width) (chroma
 * half of each) is read or written.  The call returns -1 before launching anything when a picture has mb_width / mb_height outside
 * 1..4096, mb_stride <= mb_width, a linesize below the aligned width, a NULL pointer or a chroma_qscale_table entry above 31, or when two
 * pictures of the call overlap in memory.  A qscale_table entry outside 1..31 (the decoder stores none) counts as an unfiltered macroblock. */
typedef struct FFH263LoopFilterPicture {
    uint8_t *data[3];                   /* s->current_picture.f->data (device) */
    int linesize, uvlinesize;
    int mb_width, mb_height, mb_stride;
    const uint32_t *mb_type;            /* device, s->current_picture.mb_type, indexed mb_x + mb_y * mb_stride; only IS_SKIP is read */
    const int8_t *qscale_table;         /* device, s->current_picture.qscale_table, same index */
    uint8_t chroma_qscale_table[32];    /* s->chroma_qscale_table: the default one, or ff_h263_chroma_qscale_table under Annex T */
} FFH263LoopFilterPicture;
int ff_h263_loop_filter_batch_cuda(const FFH263LoopFilterPicture *pictures /* host array */, int n_pictures, void *stream);

typedef struct FFMpvPictureWork {
    const FFMpvMCPicture *pictures; int n_pictures;     /* host array: ff_mpv_motion_batch_cuda */
    uint32_t *rejected;                                 /* device uint32, see ff_mpv_motion_batch_cuda */
    const FFMpvResidualBatch *residual; int n_residual; /* host array, run in this order after the motion compensation */
    const FFH263LoopFilterPicture *loop_filter;         /* host array, NULL / 0: none; ff_h263_loop_filter_batch_cuda after the residual */
    int n_loop_filter;
} FFMpvPictureWork;
int ff_mpv_flush_pictures_cuda(const FFMpvPictureWork *work /* host struct */, void *stream);

/* FDCTDSPContext (libavcodec/fdctdsp.h:26-29), in place over n blocks: which 0 = ff_jpeg_fdct_islow_8, 1 =
 * ff_fdct248_islow_8 (jfdctint_template.c:260-398), 2 = ff_fdct_ifast, 3 = ff_fdct_ifast248 (jfdctfst.c:207-332), 4 = ff_jpeg_fdct_islow_10,
 * 5 = ff_fdct248_islow_10 (the BIT_DEPTH 10 instances: PASS1_BITS 1, OUT_SHIFT 2; thread per block, untuned), 6 = ff_faandct, 7 = ff_faandct248
 * (libavcodec/faandct.c, bit-exact: float passes with the C code's double products; thread per block, untuned). */
int ff_fdct_batch_cuda(int which, int16_t *blocks, size_t n, void *stream);
/* PixblockDSPContext.get_pixels / diff_pixels (libavcodec/pixblockdsp_template.c:24-66) over n 8x8 blocks, optionally
 * followed by the forward DCT in the same kernel -- the encoder's "fetch (difference) -> fdct" front end
 * (mpegvideo_enc.c:1923-2019 dct loop).  Block i reads s1 + off1[i] and, if s2 != NULL, subtracts s2 + off2[i] (off2
 * NULL = the same offsets); which_fdct < 0 stores the samples / differences, 0..3, 6 and 7 select the transform as in
 * ff_fdct_batch_cuda.  Output: int16 blocks[n][64], row-major. */
int ff_pixblock_fdct_batch_cuda(int which_fdct, const uint8_t *s1, const uint8_t *s2, const uint32_t *off1, const uint32_t *off2,
                                ptrdiff_t stride, int16_t *blocks, size_t n, void *stream);

/* ---- float FFT / MDCT filterbank (FFTContext, libavcodec/fft.h:73-99); parity contract: 1e-6 relative ------------
 * ff_fft_batch_cuda: n_transforms independent complex FFTs of 2^nbits points (nbits 1..12), in place, natural order in
 * and out == the reference's fft_permute followed by fft_calc (forward kernel exp(-2 pi i jk / n), no 1/n).
 * ff_mdct_batch_cuda: op 0 imdct_half (n/2 in -> n/2 out), 1 imdct_calc (n/2 -> n), 2 mdct_calc (n -> n/2) of size
 * n = 2^nbits (4..14) with the rotation tables of ff_mdct_init(nbits, inverse, scale) (libavcodec/mdct_template.c:86-92). */
int ff_fft_batch_cuda(int nbits, int inverse, float *z, size_t n_transforms, void *stream);
int ff_mdct_batch_cuda(int op, int nbits, double scale, float *out, const float *in, size_t n_transforms, void *stream);

/* ---- libswscale boundary (libswscale/swscale.h:159-207) ------------------------------------------------
 * Same argument lists as sws_getContext / sws_scale / sws_freeContext; pixel formats are the reference's
 * AVPixelFormat values (AV_PIX_FMT_YUV420P = 0, AV_PIX_FMT_RGB24 = 2, AV_PIX_FMT_BGR24 = 3), flags the
 * reference's SWS_* bits.  Taken over: planar 8-bit yuv (420p, 422p = 4, 444p = 5, 410p = 6, 411p = 7, 440p = 31; yuva420p = 33 like 420p, src[3] is not read), gray8 = 8 (src[0] only), pal8 = 11 (src[0] indices, src[1] the 256-entry 0xAARRGGBB palette: 1024 bytes, per frame in the batch call), nv12 = 23,
 * nv21 = 24, planar 9 / 10 / 16-bit yuv 420p 422p 444p (LE and BE; scaled, or to packed destinations / another sub-sampling), and the packed yuyv422 = 1, uyvy422 = 15, rgb24, bgr24, argb / rgba / abgr / bgra (to planar yuv, or scaled to rgb24 / bgr24) sources (src[0] only) -> gray8 = 8 (the luma plane alone) / rgb24 / bgr24 / argb = 25 / rgba = 26 / abgr = 27 / bgra = 28 / rgb565 = 37 / bgr565 = 41 / rgb555 = 39 / bgr555 = 43 / rgb444 = 54 / bgr444 = 56 (and their big-endian twins 36 / 40 / 38 / 42 / 55 / 57; from planar or semi-planar yuv sources through the scaler's dithered 16-bpp output stage, output.c:869-902) / yuyv422 / uyvy422 / nv12 / nv21 (dst[0] luma, dst[1] interleaved chroma) / planar yuv (8-bit 420p
 * 422p 444p 410p 411p 440p and their full-range yuvj twins 12 / 13 / 14 / 32 on either side -- a yuv destination of the other range gets the
 * reference's range conversion, planar 8 / 9 / 10-bit only; 9 / 10 / 16-bit 420p = 62 / 64 / 47, 422p = 72 / 66 / 49, 444p = 68 / 70 / 51 little-endian and their big-endian twins), any size, SWS_FULL_CHR_H_INT or not, every scaler
 * algorithm of initFilter (libswscale/utils.c:249-632), results identical to the reference's C path under
 * SWS_ACCURATE_RND | SWS_BITEXACT.  srcFilter / dstFilter: pointers to the reference's SwsFilter (four pointers to { double *coeff; int length; }),
 * taken over for planar 8-bit yuv sources to packed rgb / planar 8-bit yuv destinations, vertical vectors symmetric.  48-bit destinations
 * rgb48be = 34 / rgb48le = 35 / bgr48be = 59 / bgr48le = 60 (yuv2rgb48_X / _2 / _1 on hScale8To19_c lines, libswscale/output.c:593-760; same size without
 * SWS_ACCURATE_RND: yuv2rgb_c_48, yuv2rgb.c:106-236) from planar 8-bit yuv / yuvj sources.  Anything else returns NULL with an error (no fallback).
 *   sws_scale_cuda         HOST pointers; whole frames (srcSliceY = 0, srcSliceH = srcH) with strides of either sign (bottom-up pictures), or
 *                          slices (not into a gray8 destination) like sws_scale() takes them (swscale_unscaled.c:1212-1340): srcSlice[] at source row srcSliceY, dst[] at the
 *                          top of the picture, top-down and contiguous, boundaries on whole chroma rows, positive strides; each call returns
 *                          (and writes) the rows the reference's loop completes with the same slices (swscale.c:483-485), at the cost of a
 *                          whole-frame pass per slice.  Uploads, runs, downloads, synchronises; returns output lines like sws_scale(),
 *                          0 on bad arguments.
 *   sws_scale_frames_cuda  DEVICE pointers, asynchronous on `stream`: nframes frames whose planes lie
 *                          *_frame_stride[] bytes apart (NULL = a single frame); returns lines written or -1.
 *                          Calls on one context must be ordered: one stream, or streams the caller synchronises.
 *                          For odd dstW the reference writes whole pixel pairs (libswscale/output.c:947); that
 *                          extra pixel is written only when dst_stride >= 3 * (dstW + 1). */
#define AVB_PIX_FMT_YUV420P 0
#define AVB_PIX_FMT_RGB24   2
#define AVB_PIX_FMT_BGR24   3
typedef struct SwsContextCUDA SwsContextCUDA;
SwsContextCUDA *sws_getContext_cuda(int srcW, int srcH, int srcFormat, int dstW, int dstH, int dstFormat, int flags,
                                    void *srcFilter, void *dstFilter, const double *param);
void sws_freeContext_cuda(SwsContextCUDA *ctx);
/* sws_setColorspaceDetails (libswscale/swscale.h:269-271, utils.c:807-835) for packed rgb destinations: inv_table = the four
 * yuv -> rgb coefficients (ff_yuv2rgb_coeffs[], e.g. SWS_CS_ITU709 = { 117504, 138453, 13954, 34903 }), srcRange 1 = full-range
 * (JPEG) yuv, brightness / contrast / saturation in 16.16 fixed point (0, 1 << 16, 1 << 16 = neutral).  Returns 0, or -1 for a yuv
 * destination (like the reference) and for settings that would index outside the reference's 1024-entry colour table.  The
 * full-range source formats yuvj420p = 12, yuvj422p = 13, yuvj444p = 14 are taken over as sources of rgb destinations. */
int sws_setColorspaceDetails_cuda(SwsContextCUDA *ctx, const int inv_table[4], int srcRange, const int table[4], int dstRange,
                                  int brightness, int contrast, int saturation);
int  sws_scale_cuda(SwsContextCUDA *ctx, const uint8_t *const srcSlice[], const int srcStride[], int srcSliceY,
                    int srcSliceH, uint8_t *const dst[], const int dstStride[]);
int  sws_scale_frames_cuda(SwsContextCUDA *ctx, const uint8_t *const src[3], const int srcStride[3],
                           const size_t srcFrameStride[3], uint8_t *const dst[3], const int dstStride[3],
                           const size_t dstFrameStride[3], int nframes, void *stream);
int  sws_is_fused_cuda(SwsContextCUDA *ctx);   /* 1 when the single-kernel same-size path is selected */
/* host-only introspection of the set-up stage (filter banks / colour constants), used to pin it against the
 * reference without a GPU: which = 0 hLum, 1 hChr, 2 vLum, 3 vChr; returns taps per output sample */
int  sws_debug_filter_cuda(int which, int srcW, int srcH, int dstW, int dstH, int dstFormat, int flags,
                           int16_t *filter, int32_t *pos, int cap, int *n_out);
/* the same with a SwsFilter pair (the reference's struct: four pointers to { double *coeff; int length; }), NULL = none */
int  sws_debug_filter2_cuda(int which, int srcW, int srcH, int dstW, int dstH, int dstFormat, int flags, const void *srcFilter,
                            const void *dstFilter, int16_t *filter, int32_t *pos, int cap, int *n_out);
void sws_debug_rgb_constants_cuda(int32_t out[10]);
/* what sws_getContext_cuda would decide, computed on the host only: 1 = taken over (out[0] path: 1 plane copy, 2 unscaled table
 * converter, 3 fused same-size kernel, 4 general scaler, 5 packed-source special converter, 6 planar -> packed 4:2:2 converter,
 * 7 yuv420p -> nv12 interleave; out[1..4] chrSrcW chrSrcH chrDstW chrDstH; out[5] source pre-pass 0 / 1 nv split / 2 reader;
 * out[6] destination bits per sample (planar) or bytes per pixel (packed); out[7] full-range source), 0 = refused */
int  sws_debug_plan_cuda(int srcW, int srcH, int srcFormat, int dstW, int dstH, int dstFormat, int flags, int32_t out[8]);
/* what the per-line slots (section 3, ff_sws_init_swscale_cuda) would know about that context: 26 int32 (19 colour constants, flags,
 * planar, destination bits, big endian, packed target, nv12 / nv21, range conversion); returns the count, 0 = refused.  Host only. */
int  sws_debug_slot_view_cuda(int srcW, int srcH, int srcFormat, int dstW, int dstH, int dstFormat, int flags, int32_t out[32]);

/* ------------------------------------------------------------------ 3. table hooks --------------- */
/* One more arch behind ff_idctdsp_init()'s dispatch (libavcodec/idctdsp.c:183-188; same shape as
 * ff_idctdsp_init_x86, libavcodec/idctdsp.h:109-110).  AVCodecContext is opaque to this library, so the
 * two fields the hook needs are passed by value (INTEGRATION.md shows the one-line caller).
 * Taken over: idct_algo FF_IDCT_SIMPLE / FF_IDCT_AUTO and FF_IDCT_FAAN (AVB_FF_IDCT_FAAN: ff_faanidct*, FF_IDCT_PERM_NONE) at 8 bit, and
 * bits_per_raw_sample 10 (ff_simple_idct_*_10 whatever idct_algo says, idctdsp.c:151-155); anything else leaves `c` untouched. */
void ff_idctdsp_init_cuda(IDCTDSPContext *c, int idct_algo, int bits_per_raw_sample, unsigned high_bit_depth);
/* The arch hook of ff_xvid_idct_init (libavcodec/xvididct.c:333-350), called after it: idct / idct_put / idct_add, perm_type =
 * FF_IDCT_PERM_NONE and an identity idct_permutation when bits_per_raw_sample <= 8 and idct_algo is FF_IDCT_AUTO or FF_IDCT_XVID
 * (AVB_FF_IDCT_XVID); otherwise `c` is untouched.  ff_idctdsp_init_cuda leaves FF_IDCT_XVID alone, like the reference's ff_idctdsp_init. */
void ff_xvid_idct_init_cuda(IDCTDSPContext *c, int idct_algo, int bits_per_raw_sample);
/* libavcodec/proresdsp.c:70-80 without the x86 part: idct_put = the slot of prores_idct_put_c (a batch of one of
 * ff_prores_idct_put_batch_cuda with host pointers), idct_permutation_type = FF_IDCT_PERM_NONE and the identity permutation. */
void ff_proresdsp_init_cuda(ProresDSPContext *dsp);
void ff_blockdsp_init_cuda(BlockDSPContext *c);   /* libavcodec/blockdsp.c:60-74 */
/* libavcodec/fdctdsp.c:27-50 (same shape as ff_fdctdsp_init_x86): dct_algo FF_DCT_AUTO / FF_DCT_INT -> islow,
 * FF_DCT_FASTINT -> ifast, FF_DCT_FAAN -> ff_faandct / ff_faandct248; bits_per_raw_sample 10 -> jpeg_fdct_islow_10 / fdct248_islow_10
 * whatever dct_algo says */
void ff_fdctdsp_init_cuda(FDCTDSPContext *c, int dct_algo, int bits_per_raw_sample, unsigned high_bit_depth);
/* libavcodec/me_cmp.c:895-944: every slot ff_me_cmp_init fills except the encoder-state metrics */
void ff_me_cmp_init_cuda(MECmpContext *c);
/* MECmpContext.quant_psnr[0..1] / bit[0..1] / rd[0..1] as slots.  They read a LIVE encoder context through `view`: host pointers to the
 * fields of the MpegEncContext `s` the C functions read (and the two they write: mb_intra, block_last_index[0]), filled once by the glue
 * with the reference's own headers (examples/reference_binding/dsp_init_cuda.c); every call snapshots them, so qscale / mb_intra may change
 * between macroblocks like in the encoder loop.  `s` is only the key the slots find their view by (struct MpegEncContext stays opaque).
 * Returns 0, or -1 (table untouched) for a state the kernels do not cover: a permuting IDCT, denoise_dct (s->dct_error_sum), trellis. */
typedef struct FFMECmpEncView {
    const int *qscale, *y_dc_scale, *h263_aic, *intra_quant_bias, *inter_quant_bias, *ac_esc_length;
    int *mb_intra, *block_last_index;
    int (*const *q_intra_matrix)[64], (*const *q_inter_matrix)[64];     /* &s->q_intra_matrix, &s->q_inter_matrix */
    const uint16_t *intra_matrix, *inter_matrix;
    const uint8_t *scantable;                                            /* s->intra_scantable.scantable */
    uint8_t *const *intra_ac_vlc_length, *const *intra_ac_vlc_last_length, *const *inter_ac_vlc_length, *const *inter_ac_vlc_last_length;
    const uint8_t *const *luma_dc_vlc_length;                            /* &s->intra_ac_vlc_length ... (codec init may set them later) */
    int fdct, dequant;                                                   /* as in FFMECmpEncState (the glue compares function pointers) */
    int idct_perm_none, plain_quantiser;                                 /* s->idsp.perm_type == FF_IDCT_PERM_NONE; fast_dct_quantize == ff_dct_quantize_c && !dct_error_sum */
} FFMECmpEncView;
int ff_me_cmp_enc_init_cuda(MECmpContext *c, struct MpegEncContext *s, const FFMECmpEncView *view);
void ff_me_cmp_enc_uninit_cuda(struct MpegEncContext *s);
/* The arch hook of the encoder's quantiser (same place as ff_mpv_encode_init_x86, libavcodec/mpegvideo_enc.c:741, :773-779): fills
 * *view->fast_dct_quantize with the plain slot and *view->dct_quantize with the trellis slot when `trellis` (avctx->trellis) is set, the
 * plain one otherwise.  The slots have the reference's signature and apply noise reduction themselves when *view->dct_error_sum is set, as the
 * C quantisers do.  Like the metric slots they read the live context through `view` on every call (one block: stage, copy, kernel, copy
 * back, synchronise).  Returns 0, or -1 with the context untouched for: a permuting IDCT, an fdct other than islow / ifast / FAAN (a
 * 10-bit encoder), quantizer_noise_shaping, slice threading (slice_context_count > 1), a NULL view pointer.  Slice threading is refused
 * because the view points into the one context it was made from: ff_update_duplicate_context copies the slots into the per-thread
 * contexts, whose mb_intra, lambda2, coded_score and noise-reduction sums are their own.  Such an encoder keeps the C quantisers (the
 * batched call serves it instead).  Call it after ff_me_cmp_enc_init_cuda, which must still see
 * fast_dct_quantize == ff_dct_quantize_c. */
typedef struct FFMpvQuantView {
    const int *mb_intra, *y_dc_scale, *c_dc_scale, *h263_aic;
    const unsigned *lambda2;
    const int *intra_quant_bias, *inter_quant_bias, *ac_esc_length, *min_qcoeff, *max_qcoeff;
    int (*const *q_intra_matrix)[64], (*const *q_inter_matrix)[64];     /* &s->q_intra_matrix, &s->q_inter_matrix */
    const uint16_t *intra_matrix, *inter_matrix;
    const uint8_t *scantable;                                            /* s->intra_scantable.scantable */
    uint8_t *const *intra_ac_vlc_length, *const *intra_ac_vlc_last_length, *const *inter_ac_vlc_length, *const *inter_ac_vlc_last_length;
    int (*const *dct_error_sum)[64];                                     /* &s->dct_error_sum (NULL inside = noise reduction off) */
    uint16_t (*const *dct_offset)[64];                                   /* &s->dct_offset */
    int *dct_count;                                                      /* s->dct_count */
    int *coded_score;                                                    /* s->coded_score */
    int (**dct_quantize)(struct MpegEncContext *, int16_t *, int, int, int *);       /* &s->dct_quantize */
    int (**fast_dct_quantize)(struct MpegEncContext *, int16_t *, int, int, int *);  /* &s->fast_dct_quantize */
    int fdct;                                                            /* 0 ff_jpeg_fdct_islow_8, 2 ff_fdct_ifast, anything else refused */
    int out_format, mpeg_quant;                                          /* s->out_format, s->mpeg_quant */
    int idct_perm_none;                                                  /* s->idsp.perm_type == FF_IDCT_PERM_NONE */
    int quantizer_noise_shaping;                                         /* s->quantizer_noise_shaping */
    int slice_context_count;                                             /* s->slice_context_count: must be 1 (see above) */
} FFMpvQuantView;
int ff_mpv_quantize_init_cuda(struct MpegEncContext *s, const FFMpvQuantView *view, int trellis);
void ff_mpv_quantize_uninit_cuda(struct MpegEncContext *s);
/* libavcodec/h264dsp.c:57-143, h264qpel.c:36-89, h264chroma.c:32-55, hpeldsp.c:338-366.  bit_depth 8, and 9 / 10 (the reference's BIT_DEPTH > 8
 * instances: uint8_t * arguments point at uint16 samples, int16_t * at int32 coefficients, strides stay in bytes).  ff_h264dsp_init_cuda fills
 * every entry ff_h264dsp_init fills (mbaff loop filters and startcode_find_candidate included); chroma_format_idc > 1 selects the
 * 4:2:2 entries (idct_add8_422, the 2x4 chroma DC transform, the 16-line h_ chroma filters) exactly like h264dsp.c:81-122 */
void ff_h264dsp_init_cuda(H264DSPContext *c, const int bit_depth, const int chroma_format_idc);
void ff_h264qpel_init_cuda(H264QpelContext *c, int bit_depth);
void ff_h264chroma_init_cuda(H264ChromaContext *c, int bit_depth);
void ff_hpeldsp_init_cuda(HpelDSPContext *c, int flags);
/* libavcodec/h264pred.h:112-123; takes over codec_id AV_CODEC_ID_H264, bit_depth 8 / 9 / 10 (16-bit samples, int32 residual above 8);
 * chroma_format_idc > 1 installs the 8 x 16 chroma functions in pred8x8[] / pred8x8_add[] like h264pred.c:477-563 */
void ff_h264_pred_init_cuda(H264PredContext *h, int codec_id, const int bit_depth, const int chroma_format_idc);
/* libavcodec/pixblockdsp.h:37-43; high_bit_depth != 0 leaves the table untouched */
void ff_pixblockdsp_init_cuda(PixblockDSPContext *c, unsigned high_bit_depth);
/* libavcodec/qpeldsp.h:75-77 */
void ff_qpeldsp_init_cuda(QpelDSPContext *c);
/* H263DSPContext (libavcodec/h263dsp.c:117-124): h263_h_loop_filter / h263_v_loop_filter as a batch of one through the picture filter's
 * line arithmetic; host pointers, the 4 x 8 samples the C function reads around src (two before it) staged and written back.  A qscale
 * outside 0..31, where the C function would read past its strength table, leaves the samples untouched. */
void ff_h263dsp_init_cuda(H263DSPContext *c);
/* MpegVideoDSPContext (libavcodec/mpegvideodsp.c:110-119): gmc1 (gmc1_c) and gmc (ff_gmc_c) as a batch of one through the GMC
 * arithmetic of ff_mpv_motion_batch_cuda; host pointers.  gmc1 stages the 9 x (h + 1) samples it reads at src; gmc stages the
 * bounding rectangle of the positions its block's four corners map to, clamped to [0, width) x [0, height) of the plane at src (the
 * whole plane where a corner leaves int32), and writes the 8 x h block back. */
void ff_mpegvideodsp_init_cuda(MpegVideoDSPContext *c);
/* libavcodec/fft_template.c:152-159, mdct_template.c:58-66 (same shape as ff_fft_init_x86 / ff_mdct_init_x86): called after
 * ff_fft_init / ff_mdct_init filled the context.  fft_permute stays the reference's; the CUDA fft_calc accepts its revtab
 * order, the MDCT slots use the context's own tcos / tsin tables. */
void ff_fft_init_cuda(FFTContext *s);
void ff_mdct_init_cuda(FFTContext *s);


/* libswscale's per-line slots: what sws_init_swscale() and its arch hooks (ff_sws_init_swscale_x86 / _ppc, libswscale/swscale.c:723-783)
 * install in a SwsContext (the function-pointer fields of libswscale/swscale_internal.h:312-330,478-535), with the reference's
 * signatures (swscale_internal.h:62-110) and HOST pointers.  `struct SwsContext` stays opaque to this library: it is only the key under
 * which ff_sws_init_swscale_cuda() remembers which SwsContextCUDA (destination format, colour constants) a slot call belongs to.
 * Filled like the reference fills them for an 8-bit source: hyScale / hcScale = hScale8To15_c (hScale8To19_c for a 16-bit destination),
 * hyscale_fast / hcscale_fast only with SWS_FAST_BILINEAR (and not for 16-bit destinations), yuv2plane1 / yuv2planeX by destination depth
 * (8, 9, 10, 16; LE / BE), yuv2nv12cX for nv12 / nv21, yuv2packed1 / 2 / X for rgb24 bgr24 argb rgba abgr bgra yuyv422 uyvy422 (only
 * yuv2packedX with SWS_FULL_CHR_H_INT, output.c:1392-1472); entries the reference leaves NULL are set to NULL.  Each call is a batch of
 * one line on the GPU (stage, copy, kernel, copy back, synchronise): plumbing and parity, like the DSP table slots -- whole frames go
 * through sws_scale_cuda / sws_scale_frames_cuda. */
struct SwsContext;
typedef struct SwsLineSlotsCUDA {
    void (*hyScale)(struct SwsContext *c, int16_t *dst, int dstW, const uint8_t *src, const int16_t *filter, const int32_t *filterPos, int filterSize);
    void (*hcScale)(struct SwsContext *c, int16_t *dst, int dstW, const uint8_t *src, const int16_t *filter, const int32_t *filterPos, int filterSize);
    void (*hyscale_fast)(struct SwsContext *c, int16_t *dst, int dstWidth, const uint8_t *src, int srcW, int xInc);
    void (*hcscale_fast)(struct SwsContext *c, int16_t *dst1, int16_t *dst2, int dstWidth, const uint8_t *src1, const uint8_t *src2, int srcW, int xInc);
    void (*yuv2plane1)(const int16_t *src, uint8_t *dest, int dstW, const uint8_t *dither, int offset);
    void (*yuv2planeX)(const int16_t *filter, int filterSize, const int16_t **src, uint8_t *dest, int dstW, const uint8_t *dither, int offset);
    void (*yuv2nv12cX)(struct SwsContext *c, const int16_t *chrFilter, int chrFilterSize, const int16_t **chrUSrc, const int16_t **chrVSrc,
                       uint8_t *dest, int dstW);
    void (*yuv2packed1)(struct SwsContext *c, const int16_t *lumSrc, const int16_t *chrUSrc[2], const int16_t *chrVSrc[2], const int16_t *alpSrc,
                        uint8_t *dest, int dstW, int uvalpha, int y);
    void (*yuv2packed2)(struct SwsContext *c, const int16_t *lumSrc[2], const int16_t *chrUSrc[2], const int16_t *chrVSrc[2],
                        const int16_t *alpSrc[2], uint8_t *dest, int dstW, int yalpha, int uvalpha, int y);
    void (*yuv2packedX)(struct SwsContext *c, const int16_t *lumFilter, const int16_t **lumSrc, int lumFilterSize, const int16_t *chrFilter,
                        const int16_t **chrUSrc, const int16_t **chrVSrc, int chrFilterSize, const int16_t **alpSrc, uint8_t *dest, int dstW, int y);
    /* set when the context converts between full-range (yuvj) and limited-range yuv (swscale.c:748-757): lum / chrRangeFromJpeg_c or
     * lum / chrRangeToJpeg_c on 15-bit lines, in place; NULL otherwise */
    void (*lumConvertRange)(int16_t *dst, int width);
    void (*chrConvertRange)(int16_t *dst1, int16_t *dst2, int width);
} SwsLineSlotsCUDA;
/* 0, or -1 (sticky error) for a NULL argument.  The registration lasts until sws_freeContext_cuda(cuda). */
int ff_sws_init_swscale_cuda(struct SwsContext *c, SwsContextCUDA *cuda, SwsLineSlotsCUDA *slots);

#ifdef __cplusplus
}
#endif
#endif /* AVDSP_B200_H */
