// libav_b200/csrc/me_cmp_enc.cu -- MECmpContext.quant_psnr / bit / rd (libavcodec/me_cmp.c:621-782, 16-wide wrappers :883-885): the three
// comparison metrics that run the encoder's quantiser on the difference of two blocks.
//
//   quant_psnr8x8_c (:621-645)  diff -> ff_dct_quantize_c as an INTER block -> dct_unquantize_inter -> ff_simple_idct_8 -> sum (rec - diff)^2
//   bit8x8_c        (:713-782)  diff -> ff_dct_quantize_c -> run / level VLC lengths (+ the DC length for an intra block)
//   rd8x8_c         (:647-711)  both: squared error of (src2 + rec) against src1 + ((bits * qscale^2 * 109 + 64) >> 7)
//
// ff_dct_quantize_c (libavcodec/mpegvideo_enc.c:4371-4450) per coefficient: level = coef * qmat[j]; a level is kept when
// (unsigned)(level + threshold1) > threshold2, as (bias +- level) >> QMAT_SHIFT with its sign; the C code's two scan-order loops (find
// the last kept position from the back, then quantise up to it) reduce to "kept or zero" per position plus the largest kept position.
// The inverse quantisers (libavcodec/mpegvideo.c:51-270) only ever change non-zero levels and every non-zero level lies inside the range
// they walk (the quantiser has just zeroed everything behind last_non_zero), so they are per-coefficient rules here too; the MPEG-2
// mismatch control needs the sum of the reconstructed levels.
//
// One thread = one record (its 1 / 2 / 4 8x8 blocks one after the other, like the wrappers); all arithmetic is thread-local (no shared
// memory, no collectives), so tests/hostsim/ runs this file on the CPU against the compiled reference.  These are encoder decision
// metrics: thousands of records per launch, instruction-bound (two transforms + two scans per block); the state lives in device memory.
#include "common.cuh"
#include "fdct_dev.cuh"
#include "mpv_quant.cuh"
#include "simple_idct8.cuh"
#include "scratch.h"
#include "../../include/avdsp_b200.h"
#include <map>
#include <mutex>
#include <string.h>

namespace avb {

struct EncDev {
    FFMECmpEncState st;
    const uint8_t *vlc[5];          // device copies: intra len, intra last, inter len, inter last, luma dc
};

// ---- device copies of the codec's VLC length tables, keyed by their host addresses (static tables in the reference) ----
// The per-call slots look the copy up by address alone; the two places a caller announces tables (ff_me_cmp_enc_init_cuda, ff_me_cmp_enc_state_cuda)
// also compare a checksum of the host bytes with the one taken at upload, so memory that was freed and reused for other tables gets a fresh copy
// (the old one stays alive for the states that point at it).
// (shared with mpv_quant.cu, declared in mpv_quant.cuh)
struct VlcKey { const uint8_t *p[5]; bool operator<(const VlcKey &o) const { return memcmp(p, o.p, sizeof(p)) < 0; } };
struct VlcCopy { uint8_t *d; uint64_t sum; };
namespace {
std::mutex g_vlc_mu;
std::map<VlcKey, VlcCopy> g_vlc;
constexpr size_t VLC_BYTES = 4 * 64 * 128 + 512;

uint64_t vlc_checksum(const VlcKey &key)
{
    uint64_t h = 0xcbf29ce484222325ull;
    for (int k = 0; k < 5; k++) {
        const size_t n = k < 4 ? 8192 : 512;
        for (size_t i = 0; i < n; i += 8) { uint64_t w; memcpy(&w, key.p[k] + i, 8); h = (h ^ w) * 0x100000001b3ull; h ^= h >> 29; }
    }
    return h;
}
}  // namespace

const uint8_t *vlc_device(const FFMECmpVlcTables *v, const char *where, bool verify)
{
    const VlcKey key = { { v->intra_ac_vlc_length, v->intra_ac_vlc_last_length, v->inter_ac_vlc_length, v->inter_ac_vlc_last_length, v->luma_dc_vlc_length } };
    for (int k = 0; k < 5; k++) if (!key.p[k]) { set_error_msg(where, "a VLC length table is NULL"); return nullptr; }
    std::lock_guard<std::mutex> lk(g_vlc_mu);
    auto it = g_vlc.find(key);
    if (it != g_vlc.end() && !verify) return it->second.d;
    const uint64_t sum = vlc_checksum(key);
    if (it != g_vlc.end() && it->second.sum == sum) return it->second.d;
    uint8_t *d = nullptr;
    if (cudaMalloc(&d, VLC_BYTES) != cudaSuccess) { set_error(where, cudaGetLastError()); return nullptr; }
    bool ok = true;
    for (int k = 0; k < 4; k++) ok = ok && cudaMemcpy(d + (size_t)k * 8192, key.p[k], 8192, cudaMemcpyHostToDevice) == cudaSuccess;
    ok = ok && cudaMemcpy(d + 4 * 8192, key.p[4], 512, cudaMemcpyHostToDevice) == cudaSuccess;
    if (!ok) { set_error(where, cudaGetLastError()); cudaFree(d); return nullptr; }
    g_vlc[key] = VlcCopy{ d, sum };
    return d;
}
namespace {

// s->fdsp.fdct on an int16 block held by the thread (int16 write-back between the passes, like fdct_kernel); fdct as in FFMECmpEncState
__device__ inline void enc_fdct(int16_t *b, int fdct)
{
    if (fdct == 6) {                                              // ff_faandct: float between the passes (fdct_dev.cuh)
        int m[8][8];
        for (int r = 0; r < 8; r++) {
            int in[8];
            for (int k = 0; k < 8; k++) in[k] = b[8 * r + k];
            fdct_row<6>(in, m[r]);
        }
        fdct_cols<6>(m);
        for (int k = 0; k < 64; k++) b[k] = (int16_t)m[k >> 3][k & 7];
        return;
    }
    const bool fast = fdct == 2;
    for (int r = 0; r < 8; r++) {
        int in[8], o[8];
        for (int k = 0; k < 8; k++) in[k] = b[8 * r + k];
        if (fast) ifast_1d(in, o); else islow_1d<4, 9>(in, o);
        for (int k = 0; k < 8; k++) b[8 * r + k] = (int16_t)o[k];
    }
    for (int c = 0; c < 8; c++) {
        int in[8], o[8];
        for (int k = 0; k < 8; k++) in[k] = b[8 * k + c];
        if (fast) ifast_1d(in, o); else islow_1d<-4, 17>(in, o);
        for (int k = 0; k < 8; k++) b[8 * k + c] = (int16_t)o[k];
    }
}

// one inverse-quantised level (mpegvideo.c:51-270); `level` != 0, j = raster position, never the DC of an intra block
__device__ __forceinline__ int enc_dequant_level(const FFMECmpEncState &S, int level, int j, bool intra)
{
    const int a = level < 0 ? -level : level;
    int v;
    if (S.dequant == 3) v = a * (S.qscale << 1) + ((intra && S.h263_aic) ? 0 : ((S.qscale - 1) | 1));
    else if (intra)     v = (a * S.qscale * (int)S.intra_matrix[j]) >> 3;
    else                v = (((a << 1) + 1) * S.qscale * (int)S.inter_matrix[j]) >> 4;
    if (S.dequant == 0) v = (v - 1) | 1;
    return level < 0 ? -v : v;
}

// the metric of one 8x8 block; `last` = ff_dct_quantize_c's return value
__device__ inline int enc_block(const EncDev &E, int kind, const uint8_t *s1, const uint8_t *s2, ptrdiff_t stride, int &last)
{
    const FFMECmpEncState &S = E.st;
    int16_t t[64], bak[64];
    for (int y = 0; y < 8; y++)
        for (int x = 0; x < 8; x++) bak[8 * y + x] = t[8 * y + x] = (int16_t)((int)s1[y * stride + x] - (int)s2[y * stride + x]);     // pdsp.diff_pixels
    const bool intra = kind != 14 && S.mb_intra != 0;            // quant_psnr clears s->mb_intra first (:629)
    // ---- ff_dct_quantize_c ----
    enc_fdct(t, S.fdct);
    int kept_or;                                                  // (unused: these metrics never clip; n = 0, a luma block, :4389-4396)
    last = mpv_quantize(t, intra, (S.h263_aic ? 1 : S.y_dc_scale) << 3, intra ? S.q_intra_matrix : S.q_inter_matrix,
                        intra ? S.intra_quant_bias : S.inter_quant_bias, S.scantable, kept_or);
    // ---- VLC bits (bit8x8_c / rd8x8_c) ----
    int bits = 0;
    if (kind != 14) {
        const uint8_t *len = E.vlc[intra ? 0 : 2], *len_last = E.vlc[intra ? 1 : 3];
        if (intra) bits = E.vlc[4][min(max((int)t[0] + 256, 0), 511)];
        int run = 0;
        for (int i = intra ? 1 : 0; i <= last; i++) {
            const int level = t[S.scantable[i]];
            if (!level && i < last) { run++; continue; }
            const unsigned idx = (unsigned)(level + 64);
            bits += idx < 128u ? (int)(i == last ? len_last : len)[run * 128 + idx] : S.ac_esc_length;
            run = 0;
        }
        if (kind == 15) return bits;
    }
    // ---- s->dct_unquantize_intra / _inter (rd8x8_c skips it for an empty block, quant_psnr8x8_c does not: the MPEG-2 inter
    //      quantiser then still toggles block[63], mpegvideo.c:199) ----
    if (kind == 14 || last >= 0) {
        int sum = -1;
        if (intra && !(S.dequant == 3 && S.h263_aic)) t[0] = (int16_t)(t[0] * S.y_dc_scale);
        for (int j = intra ? 1 : 0; j < 64; j++) {
            const int level = t[j];
            if (!level) continue;
            const int v = enc_dequant_level(S, level, j, intra);
            t[j] = (int16_t)v;
            sum += v;
        }
        if ((S.dequant == 1 && !intra) || S.dequant == 2) t[63] ^= (int16_t)(sum & 1);          // mpeg2_inter_c and mpeg2_intra_bitexact
    }
    // ---- reconstruction ----
    enc_idct_rows(t);
    int score = 0;
    for (int c = 0; c < 8; c++) {
        int o[8];
        enc_idct_col(t + c, o);
        for (int k = 0; k < 8; k++) {
            int d;
            if (kind == 14) d = (int)(int16_t)o[k] - (int)bak[8 * k + c];                       // ff_simple_idct_8 stores int16
            else d = min(max((int)s2[k * stride + c] + o[k], 0), 255) - (int)s1[k * stride + c]; // idct_add onto src2, sse against src1
            score += d * d;
        }
    }
    return kind == 14 ? score : score + ((bits * S.qscale * S.qscale * 109 + 64) >> 7);
}

__global__ void __launch_bounds__(128)
me_cmp_enc_kernel(int kind, int sidx, const EncDev *__restrict__ E, const uint8_t *__restrict__ cur, const uint8_t *__restrict__ ref, ptrdiff_t st, int h,
                  const FFMECmpRecord *__restrict__ recs, size_t n, int32_t *__restrict__ out, int32_t *__restrict__ last_index)
{
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const int nblk = sidx == 0 ? (h == 16 ? 4 : 2) : 1;
    const uint8_t *a = cur + recs[i].cur_off, *b = ref + recs[i].ref_off;
    int score = 0, last = -1;
    for (int k = 0; k < nblk; k++) {
        const ptrdiff_t off = (k & 1) * 8 + (k >> 1) * 8 * st;
        score += enc_block(*E, kind, a + off, b + off, st, last);
    }
    out[i] = score;
    if (last_index) last_index[i] = last;
}

int enc_launch(int kind, int sidx, const EncDev *E, const uint8_t *cur, const uint8_t *ref, ptrdiff_t stride, int h, const FFMECmpRecord *recs, size_t n,
               int32_t *out, int32_t *last_index, cudaStream_t st)
{
    if (!n) return 0;
    AVB_LAUNCH(me_cmp_enc_kernel, dim3((unsigned)((n + 127) / 128)), dim3(128), 0, st)(kind, sidx, E, cur, ref, stride, h, recs, n, out, last_index);
    return check_launch("ff_me_cmp_enc_batch_cuda");
}

bool state_ok(const FFMECmpEncState *s, const char *where)
{
    if (!s || (s->fdct != 0 && s->fdct != 2 && s->fdct != 6) || s->dequant < 0 || s->dequant > 3 || s->qscale < 1 || s->qscale > 31 || s->y_dc_scale < 1) {
        set_error_msg(where, "bad encoder state (fdct 0 | 2 | 6, dequant 0..3, qscale 1..31, y_dc_scale >= 1)"); return false;
    }
    uint64_t seen = 0;
    for (int i = 0; i < 64; i++) { if (s->scantable[i] > 63) { seen = 0; break; } seen |= 1ull << s->scantable[i]; }
    if (~seen) { set_error_msg(where, "scantable is not a permutation of 0..63"); return false; }
    return true;
}

void fill_vlc(EncDev &e, const uint8_t *d) { for (int k = 0; k < 5; k++) e.vlc[k] = d ? d + (size_t)k * 8192 : nullptr; }

// ---- slots ----
std::mutex g_view_mu;
std::map<const void *, FFMECmpEncView> g_views;

template <int KIND, int SIDX> int slot_enc(struct MpegEncContext *s, uint8_t *a, uint8_t *b, ptrdiff_t stride, int h)
{
    FFMECmpEncView v;
    {
        std::lock_guard<std::mutex> lk(g_view_mu);
        auto it = g_views.find(s);
        if (it == g_views.end()) { set_error_msg("me_cmp enc slot", "no FFMECmpEncView registered for this MpegEncContext"); return 0; }
        v = it->second;
    }
    EncDev e;
    memset(&e, 0, sizeof(e));
    FFMECmpEncState &S = e.st;
    S.fdct = v.fdct; S.dequant = v.dequant; S.qscale = *v.qscale; S.mb_intra = *v.mb_intra; S.y_dc_scale = *v.y_dc_scale; S.h263_aic = *v.h263_aic;
    S.intra_quant_bias = *v.intra_quant_bias; S.inter_quant_bias = *v.inter_quant_bias; S.ac_esc_length = *v.ac_esc_length;
    if (S.qscale < 1 || S.qscale > 31) { set_error_msg("me_cmp enc slot", "qscale outside 1..31"); return 0; }
    memcpy(S.q_intra_matrix, (*v.q_intra_matrix)[S.qscale], sizeof(S.q_intra_matrix));
    memcpy(S.q_inter_matrix, (*v.q_inter_matrix)[S.qscale], sizeof(S.q_inter_matrix));
    memcpy(S.intra_matrix, v.intra_matrix, sizeof(S.intra_matrix));
    memcpy(S.inter_matrix, v.inter_matrix, sizeof(S.inter_matrix));
    memcpy(S.scantable, v.scantable, 64);
    if (!state_ok(&S, "me_cmp enc slot")) return 0;
    if (KIND != 14) {
        const FFMECmpVlcTables t = { *v.intra_ac_vlc_length, *v.intra_ac_vlc_last_length, *v.inter_ac_vlc_length, *v.inter_ac_vlc_last_length, *v.luma_dc_vlc_length };
        const uint8_t *d = vlc_device(&t, "me_cmp enc slot");
        if (!d) return 0;
        fill_vlc(e, d);
    }
    ScratchLock lk;
    Scratch &P = scratch();
    constexpr size_t SP = 32, O_A = 0, O_B = 1024, O_E = 2048, O_REC = O_E + ((sizeof(EncDev) + 15) & ~(size_t)15), O_OUT = O_REC + 16, TOTAL = O_OUT + 16;
    uint8_t *hb = (uint8_t *)P.pinned2(TOTAL), *db = (uint8_t *)P.dev(10, TOTAL);
    cudaStream_t *st = P.streams();
    if (!hb || !db || !st) return 0;
    const int w = SIDX == 0 ? 16 : 8;
    for (int y = 0; y < h; y++) { memcpy(hb + O_A + SP * y, a + y * stride, w); memcpy(hb + O_B + SP * y, b + y * stride, w); }
    memcpy(hb + O_E, &e, sizeof(e));
    memset(hb + O_REC, 0, 32);
    if (cudaMemcpyAsync(db, hb, TOTAL, cudaMemcpyHostToDevice, st[0]) != cudaSuccess) { set_error("me_cmp enc slot:h2d", cudaGetLastError()); return 0; }
    if (enc_launch(KIND, SIDX, (const EncDev *)(db + O_E), db + O_A, db + O_B, SP, h, (const FFMECmpRecord *)(db + O_REC), 1, (int32_t *)(db + O_OUT),
                   (int32_t *)(db + O_OUT) + 1, st[0])) return 0;
    if (cudaMemcpyAsync(hb + O_OUT, db + O_OUT, 16, cudaMemcpyDeviceToHost, st[0]) != cudaSuccess || cudaStreamSynchronize(st[0]) != cudaSuccess) {
        set_error("me_cmp enc slot:d2h", cudaGetLastError()); return 0;
    }
    int32_t r[2];
    memcpy(r, hb + O_OUT, 8);
    if (KIND == 14) *v.mb_intra = 0;                 // the C function's side effects on the context (:629, :636)
    v.block_last_index[0] = r[1];
    return r[0];
}

}  // namespace
}  // namespace avb

using namespace avb;

extern "C" {

void *ff_me_cmp_enc_state_cuda(const FFMECmpEncState *state, const FFMECmpVlcTables *vlc)
{
    avb::enter();
    if (!state_ok(state, "ff_me_cmp_enc_state_cuda")) return nullptr;
    EncDev e;
    memset(&e, 0, sizeof(e));
    e.st = *state;
    if (vlc) {
        const uint8_t *d = vlc_device(vlc, "ff_me_cmp_enc_state_cuda", true);
        if (!d) return nullptr;
        fill_vlc(e, d);
    }
    EncDev *dev = nullptr;
    if (cudaMalloc(&dev, sizeof(EncDev)) != cudaSuccess) { set_error("ff_me_cmp_enc_state_cuda", cudaGetLastError()); return nullptr; }
    if (cudaMemcpy(dev, &e, sizeof(e), cudaMemcpyHostToDevice) != cudaSuccess) { set_error("ff_me_cmp_enc_state_cuda", cudaGetLastError()); cudaFree(dev); return nullptr; }
    return dev;
}

void ff_me_cmp_enc_state_free_cuda(void *enc_state) { avb::enter(); if (enc_state) cudaFree(enc_state); }

int ff_me_cmp_enc_batch_cuda(int kind, int sidx, const void *enc_state, const uint8_t *cur, const uint8_t *ref, ptrdiff_t stride, int h,
                             const FFMECmpRecord *recs, size_t n, int32_t *out, int32_t *last_index, void *stream)
{
    avb::enter();
    if (kind < 14 || kind > 16 || sidx < 0 || sidx > 1 || !(h == 8 || (h == 16 && sidx == 0)) || !enc_state || (n && (!cur || !ref || !recs || !out))) {
        set_error_msg("ff_me_cmp_enc_batch_cuda", "bad argument (kind 14..16, sidx 0 | 1, h 8 or 16 for sidx 0)"); return -1;
    }
    return enc_launch(kind, sidx, (const EncDev *)enc_state, cur, ref, stride, h, recs, n, out, last_index, (cudaStream_t)stream);
}

int ff_me_cmp_enc_init_cuda(MECmpContext *c, struct MpegEncContext *s, const FFMECmpEncView *view)
{
    avb::enter();
    if (!c || !s || !view) { set_error_msg("ff_me_cmp_enc_init_cuda", "NULL argument"); return -1; }
    const void *need[] = { view->qscale, view->y_dc_scale, view->h263_aic, view->intra_quant_bias, view->inter_quant_bias, view->ac_esc_length, view->mb_intra,
                           view->block_last_index, view->q_intra_matrix, view->q_inter_matrix, view->intra_matrix, view->inter_matrix, view->scantable,
                           view->intra_ac_vlc_length, view->intra_ac_vlc_last_length, view->inter_ac_vlc_length, view->inter_ac_vlc_last_length, view->luma_dc_vlc_length };
    for (const void *p : need) if (!p) { set_error_msg("ff_me_cmp_enc_init_cuda", "a view pointer is NULL"); return -1; }
    if (!view->idct_perm_none || !view->plain_quantiser || (view->fdct != 0 && view->fdct != 2 && view->fdct != 6) || view->dequant < 0 || view->dequant > 3) {
        set_error_msg("ff_me_cmp_enc_init_cuda", "not taken over: permuting IDCT, trellis / denoising quantiser or an unknown transform");
        return -1;
    }
    {   // (the tables the view points at: uploaded, or checked against their copy, now -- the per-call slots look them up by address)
        const FFMECmpVlcTables t = { *view->intra_ac_vlc_length, *view->intra_ac_vlc_last_length, *view->inter_ac_vlc_length, *view->inter_ac_vlc_last_length, *view->luma_dc_vlc_length };
        // (an encoder that has not installed its tables yet is taken as is: bit / rd refuse per call until it has)
        if (t.intra_ac_vlc_length && t.intra_ac_vlc_last_length && t.inter_ac_vlc_length && t.inter_ac_vlc_last_length && t.luma_dc_vlc_length &&
            !vlc_device(&t, "ff_me_cmp_enc_init_cuda", true)) return -1;
    }
    { std::lock_guard<std::mutex> lk(g_view_mu); g_views[s] = *view; }
    c->quant_psnr[0] = slot_enc<14, 0>; c->quant_psnr[1] = slot_enc<14, 1>;          // me_cmp.c:926-928 (SET_CMP_FUNC)
    c->bit[0] = slot_enc<15, 0>; c->bit[1] = slot_enc<15, 1>;
    c->rd[0] = slot_enc<16, 0>; c->rd[1] = slot_enc<16, 1>;
    return 0;
}

void ff_me_cmp_enc_uninit_cuda(struct MpegEncContext *s) { avb::enter(); std::lock_guard<std::mutex> lk(g_view_mu); g_views.erase(s); }

}  // extern "C"
