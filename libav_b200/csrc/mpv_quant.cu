// libav_b200/csrc/mpv_quant.cu -- the mpegvideo encoders' quantiser stage (libavcodec/mpegvideo_enc.c), batched:
//   s->dct_quantize       fdct, denoise_dct_c (:3621-3643), then ff_dct_quantize_c (:4371-4450) or dct_quantize_trellis_c (:3645-3936)
//   clip_coeffs           (:1951-1983) on a block the quantiser reports as overflowed, intra DC never clipped
//   dct_single_coeff_elimination (:1895-1949) on inter blocks, luma threshold for blocks 0-3, chroma for the rest
// One thread per block.  The front end is pixblock_fetch (fdct_dev.cuh, the kernel behind ff_pixblock_fdct_batch_cuda): the samples are
// fetched (and differenced) and transformed in registers.  The plain quantiser is mpv_quantize (mpv_quant.cuh), shared with the
// quant_psnr / bit / rd metrics.  The trellis keeps its dynamic-programming tables in shared memory in narrow types, one column per thread
// (score int32, run uint8, level int16, survivor uint8: 520 bytes a thread), and fuses the reference's coefficient loop into the search
// loop: step i of the search needs only coeff[.][i], so coeff[2][64] / coeff_count[64] shrink to the candidates of the current position
// plus those of position 0 for the inter DC re-decision.  The noise-reduction sums are reduced over the warp and added atomically.
// No barriers, no cross-thread data except that reduction: tests/hostsim/ runs this file on the CPU (one thread after the other, the sums
// added directly) against the compiled reference.
#include "common.cuh"
#include "fdct_dev.cuh"
#include "mpv_quant.cuh"
#include "scratch.h"
#include "../../include/avdsp_b200.h"
#include <math.h>
#include <map>
#include <mutex>
#include <string.h>

namespace avb {

struct QuantDev {
    FFMpvQuantState st;
    uint16_t inv_aan[64];            // ff_inv_aanscales (aandcttab.c), derived by inv_aanscales()
    const uint8_t *vlc;              // device VLC length tables (vlc_device), NULL when the state has none
};
struct QuantHandle {                 // what ff_mpv_quant_state_cuda returns: the device state and what the launcher needs on the host
    QuantDev *dev;
    int fdct;                        // FFMpvQuantState.fdct: 0 islow, 2 ifast, 6 FAAN
    bool has_vlc;
};

namespace {

constexpr int QTPB = 64;             // threads per CTA (trellis: 64 * 520 bytes of tables)
constexpr int FMT_H263 = 2;
constexpr int BEST0 = 256 * 256 * 256 * 120;

__device__ __forceinline__ int iabs(int v) { return v < 0 ? -v : v; }
__device__ __forceinline__ int wadd(int a, int b) { return (int)((unsigned)a + (unsigned)b); }          // int32 adds that wrap like gcc's
__device__ __forceinline__ int wmul(int a, int b) { return (int)((unsigned)a * (unsigned)b); }

// one thread's dynamic-programming tables: element k at p[k * QTPB] (bank-conflict free across a warp)
struct Tabs {
    int32_t *score; uint8_t *run; int16_t *level; uint8_t *surv;
};

// dct_quantize_trellis_c after the transform and noise reduction, on the thread's raster block t.  Returns last_non_zero; max as in
// mpv_quantize; score_set / coded_score = whether and what the C code writes to s->coded_score[n].
__device__ int mpv_trellis(int16_t *t, const QuantDev &Q, int qscale, bool intra, int dc_q, unsigned lambda2, const Tabs &T, int &max,
                           bool &score_set, int &coded_score)
{
    const FFMpvQuantState &S = Q.st;
    const uint8_t *scantable = S.scantable;
    const bool h263 = S.out_format == FMT_H263;
    const int lambda = (int)(lambda2 >> 1);                  // s->lambda2 >> (FF_LAMBDA_SHIFT - 6)
    const int esc_length = S.ac_esc_length;
    int qmul = qscale * 16, qadd = ((qscale - 1) | 1) * 8;
    int start_i, last_non_zero, bias = 0;
    const int32_t *qmat;
    const uint8_t *length, *last_length;
    if (intra) {
        if (S.h263_aic) qadd = 0;
        t[0] = (int16_t)((t[0] + (dc_q >> 1)) / dc_q);
        start_i = 1; last_non_zero = 0;
        qmat = S.q_intra_matrix[qscale];
        if (S.mpeg_quant || S.out_format == 0) bias = 1 << (MPV_QMAT_SHIFT - 1);
        length = Q.vlc; last_length = Q.vlc + 8192;
    } else {
        start_i = 0; last_non_zero = -1;
        qmat = S.q_inter_matrix[qscale];
        length = Q.vlc + 2 * 8192; last_length = Q.vlc + 3 * 8192;
    }
    int last_i = start_i, last_run = 0, last_level = 0, last_score = 0;
    const unsigned t1 = (1u << MPV_QMAT_SHIFT) - (unsigned)bias - 1u, t2 = t1 << 1;
    max = 0;
    score_set = false;

    for (int i = 63; i >= start_i; i--) {
        const int j = scantable[i];
        if ((unsigned)wmul(t[j], qmat[j]) + t1 > t2) { last_non_zero = i; break; }
    }
    if (last_non_zero < start_i) {
        for (int k = start_i; k < 64; k++) t[k] = 0;
        return last_non_zero;
    }

    T.score[start_i * QTPB] = 0;
    T.surv[0] = (uint8_t)start_i;
    int survivor_count = 1;
    int c0_0 = 0, cnt_0 = 0;                                // coeff[.][0], coeff_count[0]: the inter DC re-decision
    for (int i = start_i; i <= last_non_zero; i++) {
        // ---- the coefficient loop (:3723-3748) at position i ----
        const int j = scantable[i];
        int c0, cnt;
        {
            const int level = wmul(t[j], qmat[j]);
            if ((unsigned)level + t1 > t2) {
                const int m = level > 0 ? (int)((unsigned)bias + (unsigned)level) >> MPV_QMAT_SHIFT : (int)((unsigned)bias - (unsigned)level) >> MPV_QMAT_SHIFT;
                c0 = level > 0 ? m : -m;
                cnt = m < 2 ? m : 2;
                max |= m;
            } else {
                c0 = (level >> 31) | 1;
                cnt = 1;
            }
        }
        if (i == 0) { c0_0 = c0; cnt_0 = cnt; }
        // ---- the search at position i (:3761-3864) ----
        int dct_coeff = iabs(t[j]);
        if (S.fdct == 2) dct_coeff = (dct_coeff * (int)Q.inv_aan[j]) >> 12;
        const int zero_distortion = wmul(dct_coeff, dct_coeff);
        int best_score = BEST0;
        // (entry i + 1 stays unwritten in the reference when no candidate beats BEST0 -- scores wrapped past 2^31 -- and is read there:
        // cleared here, so the result is the same on every run and on both front ends)
        T.run[(i + 1) * QTPB] = 0;
        T.level[(i + 1) * QTPB] = 0;
        for (int li = 0; li < cnt; li++) {
            int level = li ? (c0 > 0 ? c0 - 1 : c0 + 1) : c0;
            const int alevel = iabs(level);
            int unquant;
            if (h263) unquant = alevel * qmul + qadd;
            else {
                if (intra) unquant = (int)(alevel * qscale * (int)S.intra_matrix[j]) >> 3;
                else unquant = (((alevel << 1) + 1) * qscale * (int)S.inter_matrix[j]) >> 4;
                unquant = ((unquant - 1) | 1) << 3;
            }
            int distortion = wadd(wmul(unquant - dct_coeff, unquant - dct_coeff), -zero_distortion);
            level += 64;
            const bool vlc = (level & ~127) == 0;
            if (!vlc) distortion = wadd(distortion, wmul(esc_length, lambda));
            for (int s = survivor_count - 1; s >= 0; s--) {
                const int sv = T.surv[s * QTPB], run = i - sv;
                int score = vlc ? wadd(distortion, wmul(length[run * 128 + level], lambda)) : distortion;
                score = wadd(score, T.score[sv * QTPB]);
                if (score < best_score) { best_score = score; T.run[(i + 1) * QTPB] = (uint8_t)run; T.level[(i + 1) * QTPB] = (int16_t)(level - 64); }
            }
            if (h263) {
                for (int s = survivor_count - 1; s >= 0; s--) {
                    const int sv = T.surv[s * QTPB], run = i - sv;
                    int score = vlc ? wadd(distortion, wmul(last_length[run * 128 + level], lambda)) : distortion;
                    score = wadd(score, T.score[sv * QTPB]);
                    if (score < last_score) { last_score = score; last_run = run; last_level = level - 64; last_i = i + 1; }
                }
            }
        }
        T.score[(i + 1) * QTPB] = best_score;
        const int bound = last_non_zero <= 27 ? best_score : wadd(best_score, lambda);
        for (; survivor_count; survivor_count--)
            if (T.score[T.surv[(survivor_count - 1) * QTPB] * QTPB] <= bound) break;
        T.surv[survivor_count++ * QTPB] = (uint8_t)(i + 1);
    }

    if (!h263) {
        last_score = BEST0;
        for (int i = T.surv[0]; i <= last_non_zero + 1; i++) {
            int score = T.score[i * QTPB];
            if (i) score = wadd(score, wmul(lambda, 2));
            if (score < last_score) { last_score = score; last_i = i; last_level = T.level[i * QTPB]; last_run = T.run[i * QTPB]; }
        }
    }
    score_set = true;
    coded_score = last_score;

    const int dc = iabs(t[0]);
    last_non_zero = last_i - 1;
    for (int k = start_i; k < 64; k++) t[k] = 0;
    if (last_non_zero < start_i) return last_non_zero;

    if (last_non_zero == 0 && start_i == 0) {                // (:3891-3923)
        int best_level = 0, best_score = wmul(dc, dc);
        for (int li = 0; li < cnt_0; li++) {
            int level = li ? (c0_0 > 0 ? c0_0 - 1 : c0_0 + 1) : c0_0;
            const int alevel = iabs(level);
            int unquant;
            if (h263) unquant = (alevel * qmul + qadd) >> 3;
            else unquant = (((((alevel << 1) + 1) * qscale * (int)S.inter_matrix[0]) >> 4) - 1) | 1;
            unquant = ((unquant + 4) >> 3) << 6;
            const int distortion = wmul(unquant - dc, unquant - dc);
            level += 64;
            const int score = (level & ~127) == 0 ? wadd(distortion, wmul(last_length[level], lambda)) : wadd(distortion, wmul(esc_length, lambda));
            if (score < best_score) { best_score = score; best_level = level - 64; }
        }
        t[0] = (int16_t)best_level;
        coded_score = wadd(best_score, -wmul(dc, dc));
        return best_level == 0 ? -1 : last_non_zero;
    }

    t[scantable[last_non_zero]] = (int16_t)last_level;
    for (int i = last_i - last_run - 1; i > start_i; i -= T.run[i * QTPB] + 1)
        t[scantable[i - 1]] = T.level[i * QTPB];
    return last_non_zero;
}

// clip_coeffs (:1951-1983): scan positions start_i..last
__device__ __forceinline__ void mpv_clip(int16_t *t, const FFMpvQuantState &S, bool intra, int last)
{
    for (int i = intra ? 1 : 0; i <= last; i++) {
        const int j = S.scantable[i];
        int level = t[j];
        if (level > S.max_qcoeff) level = S.max_qcoeff;
        else if (level < S.min_qcoeff) level = S.min_qcoeff;
        t[j] = (int16_t)level;
    }
}

// dct_single_coeff_elimination (:1895-1949); returns the new last index
__device__ __forceinline__ int mpv_eliminate(int16_t *t, const uint8_t *scantable, int last, int threshold)
{
    const bool skip_dc = threshold >= 0;
    if (!skip_dc) threshold = -threshold;
    if (last <= (skip_dc ? 0 : -1)) return last;
    int score = 0, run = 0;
    for (int i = 0; i <= last; i++) {
        const int level = iabs(t[scantable[i]]);
        if (level == 1) {
            if (skip_dc && i == 0) continue;
            score += run == 0 ? 3 : run < 3 ? 2 : run < 24 ? 1 : 0;     // tab[run] (:1898-1907)
            run = 0;
        } else if (level > 1) return last;
        else run++;
    }
    if (score >= threshold) return last;
    for (int i = skip_dc ? 1 : 0; i <= last; i++) t[scantable[i]] = 0;
    return t[0] ? 0 : -1;
}

// noise-reduction sums: add v to *p from every lane (hostsim: the threads run one after the other)
__device__ __forceinline__ void nr_add(int32_t *p, int v)
{
#ifdef AVB_HOSTSIM
    *p += v;
#else
    v = __reduce_add_sync(0xffffffffu, v);
    if ((threadIdx.x & 31) == 0 && v) atomicAdd(p, v);
#endif
}

// POST: clip and elimination (the batch call); the slots stop after the quantiser like s->dct_quantize.
// Every lane of a warp reaches the noise-reduction reduction (no early return before it).
template <int FDCT, bool TRELLIS>
__global__ void __launch_bounds__(QTPB)
mpv_quant_kernel(const QuantDev *__restrict__ Q, const FFMpvQuantRecord *__restrict__ recs, const uint8_t *__restrict__ s1,
                 const uint8_t *__restrict__ s2, const uint32_t *__restrict__ off1, const uint32_t *__restrict__ off2, ptrdiff_t stride,
                 int16_t *__restrict__ blocks, size_t n, int32_t *__restrict__ last_index, int32_t *__restrict__ coded_score,
                 const uint16_t *__restrict__ nr_offset, int32_t *nr_sum, int32_t *nr_count, bool post)
{
    const size_t bi = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    const FFMpvQuantState &S = Q->st;
    FFMpvQuantRecord r = {};
    if (bi < n) r = recs[bi];
    const bool intra = r.intra != 0;
    const bool ok = bi < n && r.qscale >= 1 && r.qscale <= 31 && (!intra || S.h263_aic || r.dc_scale);
    int16_t t[64];
    if (ok) {
        int m[8][8];
        if (s1) pixblock_fetch<FDCT>(s1 + off1[bi], s2 ? s2 + (off2 ? off2[bi] : off1[bi]) : nullptr, stride, m);
        else fdct_load<FDCT>(blocks + 64 * bi, m);
#pragma unroll
        for (int k = 0; k < 64; k++) t[k] = (int16_t)m[k >> 3][k & 7];
    }
    if (nr_sum) {                                            // denoise_dct_c: the sums take the magnitude before the subtraction
        const uint16_t *off = nr_offset + (intra ? 64 : 0);
        nr_add(nr_count + 1, ok && intra);
        nr_add(nr_count, ok && !intra);
        for (int k = 0; k < 64; k++) {
            const int level = ok ? t[k] : 0;
            nr_add(nr_sum + 64 + k, intra ? iabs(level) : 0);
            nr_add(nr_sum + k, intra ? 0 : iabs(level));
            if (level > 0) t[k] = (int16_t)(level - (int)off[k] < 0 ? 0 : level - (int)off[k]);
            else if (level < 0) t[k] = (int16_t)(level + (int)off[k] > 0 ? 0 : level + (int)off[k]);
        }
    }
    if (!ok) return;

    const int dc_q = (S.h263_aic ? 1 : r.dc_scale) << 3;
    int max, last;
    bool score_set = false;
    int score = 0;
    if (TRELLIS) {
        __shared__ int32_t sh_score[65 * QTPB];
        __shared__ int16_t sh_level[65 * QTPB];
        __shared__ uint8_t sh_run[65 * QTPB], sh_surv[65 * QTPB];
        const int c = threadIdx.x;
        const Tabs T = { sh_score + c, sh_run + c, sh_level + c, sh_surv + c };
        last = mpv_trellis(t, *Q, r.qscale, intra, dc_q, r.lambda2, T, max, score_set, score);
    } else {
        last = mpv_quantize(t, intra, dc_q, intra ? S.q_intra_matrix[r.qscale] : S.q_inter_matrix[r.qscale],
                            intra ? S.intra_quant_bias : S.inter_quant_bias, S.scantable, max);
    }
    if (post) {
        if (S.max_qcoeff < max) mpv_clip(t, S, intra, last);
        const int thr = r.chroma ? S.chroma_elim_threshold : S.luma_elim_threshold;
        if (thr && !intra) last = mpv_eliminate(t, S.scantable, last, thr);
    } else last = (last + 1) | (S.max_qcoeff < max) << 8 | score_set << 9;   // the slot's packing: last_non_zero + 1, overflow, score written
    int16_t *d = blocks + 64 * bi;
#pragma unroll
    for (int k = 0; k < 8; k++)
        reinterpret_cast<uint4 *>(d)[k] = make_uint4(pack16(t[8 * k], t[8 * k + 1]), pack16(t[8 * k + 2], t[8 * k + 3]),
                                                     pack16(t[8 * k + 4], t[8 * k + 5]), pack16(t[8 * k + 6], t[8 * k + 7]));
    last_index[bi] = last;
    if (coded_score && score_set) coded_score[bi] = score;
}

// ff_inv_aanscales (libavcodec/aandcttab.c): 4096 / (a(u) a(v)) rounded, a(0) = 1, a(k) = sqrt(2) cos(k pi / 16)
void inv_aanscales(uint16_t *out)
{
    const double pi = 3.14159265358979323846;
    for (int i = 0; i < 64; i++) {
        const int u = i >> 3, v = i & 7;
        const double au = u ? sqrt(2.0) * cos(u * pi / 16) : 1.0, av = v ? sqrt(2.0) * cos(v * pi / 16) : 1.0;
        out[i] = (uint16_t)floor(4096.0 / (au * av) + 0.5);
    }
}

bool state_ok(const FFMpvQuantState *s, const char *where)
{
    if (!s || (s->fdct != 0 && s->fdct != 2 && s->fdct != 6) || s->out_format < 0 || s->out_format > 3) {
        set_error_msg(where, "bad quantiser state (fdct 0 | 2 | 6, out_format 0..3)"); return false;
    }
    uint64_t seen = 0;
    for (int i = 0; i < 64; i++) { if (s->scantable[i] > 63) { seen = 0; break; } seen |= 1ull << s->scantable[i]; }
    if (~seen || s->scantable[0]) { set_error_msg(where, "scantable is not a permutation of 0..63 starting at 0"); return false; }
    return true;
}

// the device tables for a state; NULL vlc = none (plain quantiser only).  The luma DC table is not read: a NULL one is replaced by zeros
// so that the shared cache, which wants all five, can hold the four AC tables of an MPEG-1 / MPEG-2 encoder.
const uint8_t *trellis_vlc(const FFMECmpVlcTables *vlc, const char *where, bool verify)
{
    static const uint8_t no_dc[512] = {};
    FFMECmpVlcTables v = *vlc;
    if (!v.luma_dc_vlc_length) v.luma_dc_vlc_length = no_dc;
    return vlc_device(&v, where, verify);
}

bool make_dev(QuantDev &q, const FFMpvQuantState *st, const FFMECmpVlcTables *vlc, const char *where, bool verify)
{
    memset(&q, 0, sizeof(q));
    if (!state_ok(st, where)) return false;
    q.st = *st;
    inv_aanscales(q.inv_aan);
    if (vlc && !(q.vlc = trellis_vlc(vlc, where, verify))) return false;
    return true;
}

int quant_launch(const QuantDev *Q, int fdct, bool trellis, const FFMpvQuantRecord *recs, const uint8_t *s1, const uint8_t *s2, const uint32_t *off1,
                 const uint32_t *off2, ptrdiff_t stride, int16_t *blocks, size_t n, int32_t *last_index, int32_t *coded_score,
                 const FFMpvNoiseReduction *nr, bool post, cudaStream_t st, const char *where)
{
    const dim3 grid((unsigned)((n + QTPB - 1) / QTPB)), block(QTPB);
    const uint16_t *o = nr ? nr->dct_offset : nullptr;
    int32_t *es = nr ? nr->dct_error_sum : nullptr, *ec = nr ? nr->dct_count : nullptr;
#define QL(F, T) AVB_LAUNCH((mpv_quant_kernel<F, T>), grid, block, 0, st)(Q, recs, s1, s2, off1, off2, stride, blocks, n, last_index, coded_score, o, es, ec, post)
    if (fdct == 2)      { if (trellis) QL(2, true); else QL(2, false); }
    else if (fdct == 6) { if (trellis) QL(6, true); else QL(6, false); }
    else                { if (trellis) QL(0, true); else QL(0, false); }
#undef QL
    return check_launch(where);
}

// ---- slots ----
std::mutex g_view_mu;
std::map<const void *, FFMpvQuantView> g_views;

template <bool TRELLIS> int slot_quant(struct MpegEncContext *s, int16_t *block, int n, int qscale, int *overflow)
{
    static const char *where = "mpv dct_quantize slot";
    FFMpvQuantView v;
    {
        std::lock_guard<std::mutex> lk(g_view_mu);
        auto it = g_views.find(s);
        if (it == g_views.end()) { set_error_msg(where, "no FFMpvQuantView registered for this MpegEncContext"); *overflow = 0; return -1; }
        v = it->second;
    }
    *overflow = 0;
    if (qscale < 1 || qscale > 31) { set_error_msg(where, "qscale outside 1..31"); return -1; }
    const bool intra = *v.mb_intra != 0;
    const int dc_scale = n < 4 ? *v.y_dc_scale : *v.c_dc_scale;
    if (intra && !*v.h263_aic && (dc_scale < 1 || dc_scale > 255)) { set_error_msg(where, "dc_scale outside 1..255"); return -1; }
    ScratchLock lk;
    Scratch &P = scratch();
    constexpr size_t O_Q = 0, O_BLK = (sizeof(QuantDev) + 15) & ~(size_t)15, O_REC = O_BLK + 128, O_NR = O_REC + 16,
                     O_OFF = O_NR + 2 * 64 * 4 + 16, O_OUT = O_OFF + 2 * 64 * 2, TOTAL = O_OUT + 16;
    uint8_t *hb = (uint8_t *)P.pinned2(TOTAL), *db = (uint8_t *)P.dev(11, TOTAL);
    cudaStream_t *st = P.streams();
    if (!hb || !db || !st) { set_error_msg(where, "no scratch memory"); return -1; }
    QuantDev &q = *(QuantDev *)(hb + O_Q);
    memset(&q, 0, sizeof(q));
    FFMpvQuantState &S = q.st;
    S.fdct = v.fdct; S.out_format = v.out_format; S.mpeg_quant = v.mpeg_quant; S.h263_aic = *v.h263_aic;
    S.intra_quant_bias = *v.intra_quant_bias; S.inter_quant_bias = *v.inter_quant_bias; S.ac_esc_length = *v.ac_esc_length;
    S.min_qcoeff = *v.min_qcoeff; S.max_qcoeff = *v.max_qcoeff;
    memcpy(S.q_intra_matrix[qscale], (*v.q_intra_matrix)[qscale], sizeof(S.q_intra_matrix[0]));
    memcpy(S.q_inter_matrix[qscale], (*v.q_inter_matrix)[qscale], sizeof(S.q_inter_matrix[0]));
    memcpy(S.intra_matrix, v.intra_matrix, sizeof(S.intra_matrix));
    memcpy(S.inter_matrix, v.inter_matrix, sizeof(S.inter_matrix));
    memcpy(S.scantable, v.scantable, 64);
    if (!state_ok(&S, where)) return -1;
    inv_aanscales(q.inv_aan);
    if (TRELLIS) {
        const FFMECmpVlcTables t = { *v.intra_ac_vlc_length, *v.intra_ac_vlc_last_length, *v.inter_ac_vlc_length, *v.inter_ac_vlc_last_length, nullptr };
        if (!(q.vlc = trellis_vlc(&t, where, false))) return -1;
    }
    memcpy(hb + O_BLK, block, 128);
    FFMpvQuantRecord rec = { (uint8_t)qscale, (uint8_t)intra, (uint8_t)dc_scale, (uint8_t)(n >= 4), *v.lambda2 };
    memcpy(hb + O_REC, &rec, sizeof(rec));
    int (*const es)[64] = *v.dct_error_sum;
    if (es) {
        memcpy(hb + O_NR, es, 2 * 64 * 4);
        memcpy(hb + O_NR + 2 * 64 * 4, v.dct_count, 8);
        memcpy(hb + O_OFF, *v.dct_offset, 2 * 64 * 2);
    }
    if (cudaMemcpyAsync(db, hb, TOTAL, cudaMemcpyHostToDevice, st[0]) != cudaSuccess) { set_error("mpv dct_quantize slot:h2d", cudaGetLastError()); return -1; }
    const FFMpvNoiseReduction nr = { (const uint16_t *)(db + O_OFF), (int32_t *)(db + O_NR), (int32_t *)(db + O_NR + 2 * 64 * 4) };
    if (quant_launch((const QuantDev *)(db + O_Q), v.fdct, TRELLIS, (const FFMpvQuantRecord *)(db + O_REC), nullptr, nullptr, nullptr, nullptr, 0,
                     (int16_t *)(db + O_BLK), 1, (int32_t *)(db + O_OUT), (int32_t *)(db + O_OUT) + 1, es ? &nr : nullptr, false, st[0], where)) return -1;
    if (cudaMemcpyAsync(hb + O_BLK, db + O_BLK, TOTAL - O_BLK, cudaMemcpyDeviceToHost, st[0]) != cudaSuccess || cudaStreamSynchronize(st[0]) != cudaSuccess) {
        set_error("mpv dct_quantize slot:d2h", cudaGetLastError()); return -1;
    }
    memcpy(block, hb + O_BLK, 128);
    if (es) {
        memcpy(es, hb + O_NR, 2 * 64 * 4);
        memcpy(v.dct_count, hb + O_NR + 2 * 64 * 4, 8);
    }
    int32_t out[2];
    memcpy(out, hb + O_OUT, 8);
    if (out[0] & 512) v.coded_score[n] = out[1];
    *overflow = (out[0] >> 8) & 1;
    return (out[0] & 255) - 1;
}

}  // namespace
}  // namespace avb

using namespace avb;

extern "C" {

void *ff_mpv_quant_state_cuda(const FFMpvQuantState *state, const FFMECmpVlcTables *vlc)
{
    avb::enter();
    QuantDev q;
    if (!make_dev(q, state, vlc, "ff_mpv_quant_state_cuda", true)) return nullptr;
    QuantHandle *h = new QuantHandle{ nullptr, state->fdct, vlc != nullptr };
    if (cudaMalloc(&h->dev, sizeof(QuantDev)) != cudaSuccess) { set_error("ff_mpv_quant_state_cuda", cudaGetLastError()); delete h; return nullptr; }
    if (cudaMemcpy(h->dev, &q, sizeof(q), cudaMemcpyHostToDevice) != cudaSuccess) {
        set_error("ff_mpv_quant_state_cuda", cudaGetLastError()); cudaFree(h->dev); delete h; return nullptr;
    }
    return h;
}

void ff_mpv_quant_state_free_cuda(void *quant_state)
{
    avb::enter();
    QuantHandle *h = (QuantHandle *)quant_state;
    if (h) { cudaFree(h->dev); delete h; }
}

int ff_mpv_dct_quantize_batch_cuda(const void *quant_state, int trellis, const FFMpvQuantRecord *recs, const uint8_t *s1, const uint8_t *s2,
                                   const uint32_t *off1, const uint32_t *off2, ptrdiff_t stride, int16_t *blocks, size_t n,
                                   int32_t *last_index, int32_t *coded_score, const FFMpvNoiseReduction *nr, void *stream)
{
    avb::enter();
    static const char *where = "ff_mpv_dct_quantize_batch_cuda";
    const QuantHandle *h = (const QuantHandle *)quant_state;
    if (!h) { set_error_msg(where, "no quantiser state"); return -1; }
    if (trellis && !h->has_vlc) { set_error_msg(where, "trellis needs a state made with VLC length tables"); return -1; }
    if (!n) return 0;
    if (!recs || !blocks || !last_index || (s1 && !off1) || (nr && (!nr->dct_offset || !nr->dct_error_sum || !nr->dct_count))) {
        set_error_msg(where, "a NULL buffer (recs, blocks, last_index; off1 with s1; the three noise-reduction arrays)"); return -1;
    }
    if ((uintptr_t)blocks & 15) { set_error_msg(where, "blocks must be 16-byte aligned"); return -1; }
    return quant_launch(h->dev, h->fdct, trellis != 0, recs, s1, s2, off1, off2, stride, blocks, n, last_index, coded_score, nr, true, (cudaStream_t)stream, where);
}

int ff_mpv_quantize_init_cuda(struct MpegEncContext *s, const FFMpvQuantView *view, int trellis)
{
    avb::enter();
    static const char *where = "ff_mpv_quantize_init_cuda";
    if (!s || !view) { set_error_msg(where, "NULL argument"); return -1; }
    const void *need[] = { view->mb_intra, view->y_dc_scale, view->c_dc_scale, view->h263_aic, view->lambda2, view->intra_quant_bias, view->inter_quant_bias,
                           view->ac_esc_length, view->min_qcoeff, view->max_qcoeff, view->q_intra_matrix, view->q_inter_matrix, view->intra_matrix,
                           view->inter_matrix, view->scantable, view->intra_ac_vlc_length, view->intra_ac_vlc_last_length, view->inter_ac_vlc_length,
                           view->inter_ac_vlc_last_length, view->dct_error_sum, view->dct_offset, view->dct_count, view->coded_score,
                           (const void *)view->dct_quantize, (const void *)view->fast_dct_quantize };
    for (const void *p : need) if (!p) { set_error_msg(where, "a view pointer is NULL"); return -1; }
    if (!view->idct_perm_none || (view->fdct != 0 && view->fdct != 2 && view->fdct != 6) || view->quantizer_noise_shaping || view->out_format < 0 || view->out_format > 3 ||
        view->slice_context_count != 1) {
        // (slice threading: the per-thread contexts are copies of `s` that carry the slots but not this view -- their own mb_intra,
        //  lambda2, coded_score and noise-reduction sums would be neither found nor used)
        set_error_msg(where, "not taken over: permuting IDCT, 10-bit transform, quantizer_noise_shaping, slice threading");
        return -1;
    }
    {   // the tables the view points at: uploaded, or checked against their copy, now -- the trellis slot looks them up by address
        // (an encoder that has not installed its tables yet is taken as is: the trellis slot refuses per call until it has)
        const FFMECmpVlcTables t = { *view->intra_ac_vlc_length, *view->intra_ac_vlc_last_length, *view->inter_ac_vlc_length, *view->inter_ac_vlc_last_length, nullptr };
        if (trellis && t.intra_ac_vlc_length && t.intra_ac_vlc_last_length && t.inter_ac_vlc_length && t.inter_ac_vlc_last_length &&
            !trellis_vlc(&t, where, true)) return -1;
    }
    { std::lock_guard<std::mutex> lk(g_view_mu); g_views[s] = *view; }
    *view->fast_dct_quantize = slot_quant<false>;               // mpegvideo_enc.c:773-779
    *view->dct_quantize = trellis ? slot_quant<true> : slot_quant<false>;
    return 0;
}

void ff_mpv_quantize_uninit_cuda(struct MpegEncContext *s) { avb::enter(); std::lock_guard<std::mutex> lk(g_view_mu); g_views.erase(s); }

}  // extern "C"
