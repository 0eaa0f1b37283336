/*
 * oracle/port/orc_mpvq.c -- TEST INFRASTRUCTURE, NOT PRODUCT.
 *
 * Plain-C restatement of the mpegvideo encoders' quantiser stage (libavcodec/mpegvideo_enc.c): the forward DCT, noise reduction
 * (denoise_dct_c), the plain quantiser (ff_dct_quantize_c) or the rate-distortion trellis (dct_quantize_trellis_c), then, per block as
 * encode_mb_internal runs them, clip_coeffs and dct_single_coeff_elimination.  Called like ref_mpvq_batch (oracle/refbuild/refapi_mpvq.c);
 * the CPU suite pins one against the other, and the GPU tests use this one where the reference was not built.  Compiled with -fwrapv:
 * the int32 products and sums wrap like the reference's code does under gcc.
 */
#include <math.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

void orc_fdct(int which, int16_t *block);                   /* orc_idct.c: 0 jpeg_fdct_islow_8, 2 fdct_ifast */

typedef struct MpvqState {
    int32_t fdct, out_format, mpeg_quant, h263_aic, intra_quant_bias, inter_quant_bias, ac_esc_length, min_qcoeff, max_qcoeff;
    int32_t luma_elim_threshold, chroma_elim_threshold;
    int32_t q_intra_matrix[32][64], q_inter_matrix[32][64];
    uint16_t intra_matrix[64], inter_matrix[64];
    uint8_t scantable[64];
    uint8_t pad[8];
} MpvqState;
typedef struct MpvqRecord { uint8_t qscale, intra, dc_scale, chroma; uint32_t lambda2; } MpvqRecord;

enum { SHIFT = 22, BIAS_UNIT_SHIFT = 8, H263 = 2, MPEG1 = 0, NO_SCORE = 256 * 256 * 256 * 120 };

/* 4096 / (a(u) a(v)) rounded to the nearest integer, a(0) = 1, a(k) = sqrt(2) cos(k pi / 16): the AAN output scale the fast FDCT leaves in */
void orc_mpvq_inv_aanscales(uint16_t *out)
{
    for (int i = 0; i < 64; i++) {
        const double a = (i >> 3) ? sqrt(2.0) * cos((i >> 3) * M_PI / 16) : 1.0, b = (i & 7) ? sqrt(2.0) * cos((i & 7) * M_PI / 16) : 1.0;
        out[i] = (uint16_t)floor(4096.0 / (a * b) + 0.5);
    }
}

static int iabs(int v) { return v < 0 ? -v : v; }

/* what the trellis tables hold before a block: the reference leaves them uninitialised, and with scores that wrap past 2^31 it can read an
 * entry it never wrote (a position where no candidate beat the initial best score).  Tests run the port with two fillings to find the blocks
 * whose result depends on that, and leave them out of every comparison. */
static int table_fill;
void orc_mpvq_set_table_fill(int v) { table_fill = v; }

/* magnitude threshold test and biased rounding of one coefficient: returns 1 when it survives, with *mag its quantised magnitude */
static int quant_one(int coef, int qm, int bias, int *mag, int *product)
{
    const int p = coef * qm;
    const unsigned thr = (1u << SHIFT) - (unsigned)bias - 1u;
    *product = p;
    if ((unsigned)(p + (int)thr) <= thr * 2u) return 0;
    *mag = p > 0 ? (bias + p) >> SHIFT : (bias - p) >> SHIFT;
    return 1;
}

static int plain_quant(const MpvqState *st, int16_t *b, int qscale, int intra, int *ovf)
{
    const int *qm = intra ? st->q_intra_matrix[qscale] : st->q_inter_matrix[qscale];
    const int bias = (intra ? st->intra_quant_bias : st->inter_quant_bias) * (1 << (SHIFT - BIAS_UNIT_SHIFT));
    int last = intra ? 0 : -1, maxmag = 0;
    for (int i = intra; i < 64; i++) {
        const int j = st->scantable[i];
        int mag, p;
        if (quant_one(b[j], qm[j], bias, &mag, &p)) {
            b[j] = p > 0 ? mag : -mag;
            maxmag |= mag;
            last = i;
        } else
            b[j] = 0;
    }
    *ovf = st->max_qcoeff < maxmag;
    return last;
}

/* the inverse quantiser the trellis weighs a candidate level with, in the FDCT's scale (<< 3) */
static int recon(const MpvqState *st, int alevel, int j, int qscale, int intra, int qmul, int qadd)
{
    int v;
    if (st->out_format == H263) return alevel * qmul + qadd;
    v = intra ? (alevel * qscale * st->intra_matrix[j]) >> 3 : (((alevel << 1) + 1) * qscale * st->inter_matrix[j]) >> 4;
    return ((v - 1) | 1) << 3;
}

static int trellis_quant(const MpvqState *st, const uint8_t *const *vlc, const uint16_t *inv_aan, int16_t *b, int qscale, int intra,
                         unsigned lambda2, int *ovf, int *coded_score)
{
    const int lambda = (int)(lambda2 >> 1), h263 = st->out_format == H263, first = intra ? 1 : 0;
    const int *qm = intra ? st->q_intra_matrix[qscale] : st->q_inter_matrix[qscale];
    const uint8_t *len = vlc[intra ? 0 : 2], *len_last = vlc[intra ? 1 : 3];
    const int bias = intra && (st->mpeg_quant || st->out_format == MPEG1) ? 1 << (SHIFT - 1) : 0;
    const int qmul = qscale * 16, qadd = intra && st->h263_aic ? 0 : ((qscale - 1) | 1) * 8;
    int cand[64][2], ncand[64], score[65], run_of[65], level_of[65], surv[65], nsurv = 1;
    int end = first - 1, maxmag = 0, end_run = 0, end_level = 0, end_score = 0, end_pos = first;
    for (int i = 0; i < 65; i++) score[i] = run_of[i] = level_of[i] = table_fill;

    for (int i = 63; i >= first; i--) {
        int mag, p;
        if (quant_one(b[st->scantable[i]], qm[st->scantable[i]], bias, &mag, &p)) { end = i; break; }
    }
    for (int i = first; i <= end; i++) {
        int mag, p;
        if (quant_one(b[st->scantable[i]], qm[st->scantable[i]], bias, &mag, &p)) {
            cand[i][0] = p > 0 ? mag : -mag;
            cand[i][1] = p > 0 ? mag - 1 : 1 - mag;
            ncand[i] = mag < 2 ? mag : 2;
            maxmag |= mag;
        } else {
            cand[i][0] = p < 0 ? -1 : 1;
            ncand[i] = 1;
        }
    }
    *ovf = st->max_qcoeff < maxmag;
    if (end < first) {
        memset(b + first, 0, (64 - first) * sizeof(*b));
        return end;
    }

    score[first] = 0;
    surv[0] = first;
    for (int i = first; i <= end; i++) {
        const int j = st->scantable[i];
        int c = iabs(b[j]), best = NO_SCORE;
        if (st->fdct == 2) c = (c * inv_aan[j]) >> 12;
        for (int k = 0; k < ncand[i]; k++) {
            const int lv = cand[i][k], u = recon(st, iabs(lv), j, qscale, intra, qmul, qadd);
            const int coded = (unsigned)(lv + 64) < 128;                  /* -64 <= lv <= 63: a table code, else an escape */
            const int dist = (u - c) * (u - c) - c * c + (coded ? 0 : st->ac_esc_length * lambda);
            for (int s = nsurv - 1; s >= 0; s--) {
                const int run = i - surv[s];
                const int sc = dist + (coded ? len[run * 128 + lv + 64] * lambda : 0) + score[surv[s]];
                if (sc < best) { best = sc; run_of[i + 1] = run; level_of[i + 1] = lv; }
            }
            if (h263)
                for (int s = nsurv - 1; s >= 0; s--) {
                    const int run = i - surv[s];
                    const int sc = dist + (coded ? len_last[run * 128 + lv + 64] * lambda : 0) + score[surv[s]];
                    if (sc < end_score) { end_score = sc; end_run = run; end_level = lv; end_pos = i + 1; }
                }
        }
        score[i + 1] = best;
        while (nsurv && score[surv[nsurv - 1]] > (end <= 27 ? best : best + lambda)) nsurv--;
        surv[nsurv++] = i + 1;
    }
    if (!h263) {
        end_score = NO_SCORE;
        for (int i = surv[0]; i <= end + 1; i++) {
            const int sc = score[i] + (i ? 2 * lambda : 0);
            if (sc < end_score) { end_score = sc; end_pos = i; end_level = level_of[i]; end_run = run_of[i]; }
        }
    }
    *coded_score = end_score;

    const int dc = iabs(b[0]);
    memset(b + first, 0, (64 - first) * sizeof(*b));
    end = end_pos - 1;
    if (end < first) return end;
    if (end == 0 && first == 0) {                       /* one inter coefficient, at DC: re-decide it against dropping the block */
        int best_lv = 0, best = dc * dc;
        for (int k = 0; k < ncand[0]; k++) {
            const int lv = cand[0][k];
            int u = h263 ? (iabs(lv) * qmul + qadd) >> 3 : (((((iabs(lv) << 1) + 1) * qscale * st->inter_matrix[0]) >> 4) - 1) | 1;
            u = ((u + 4) >> 3) << 6;
            const int sc = (u - dc) * (u - dc) + ((unsigned)(lv + 64) < 128 ? len_last[lv + 64] : st->ac_esc_length) * lambda;
            if (sc < best) { best = sc; best_lv = lv; }
        }
        b[0] = best_lv;
        *coded_score = best - dc * dc;
        return best_lv ? end : -1;
    }
    b[st->scantable[end]] = end_level;
    for (int i = end_pos - end_run - 1; i > first; i -= run_of[i] + 1)
        b[st->scantable[i - 1]] = level_of[i];
    return end;
}

int orc_mpvq_batch(const MpvqState *st, const uint8_t *const *vlc, int trellis, int post, const MpvqRecord *recs, size_t n,
                   int16_t *blocks, int32_t *last_index, int32_t *overflow, int32_t *coded_score,
                   const uint16_t *nr_offset, int32_t *nr_sum, int32_t *nr_count)
{
    uint16_t inv_aan[64];
    if (st->fdct != 0 && st->fdct != 2) return -1;
    if (trellis && !vlc) return -1;
    orc_mpvq_inv_aanscales(inv_aan);
    for (size_t k = 0; k < n; k++) {
        const MpvqRecord *r = &recs[k];
        int16_t *b = blocks + 64 * k;
        int ovf = 0, last;
        orc_fdct(st->fdct, b);
        if (nr_sum) {                                   /* noise reduction: shrink each level towards 0 by its offset */
            int32_t *sum = nr_sum + 64 * r->intra;
            const uint16_t *off = nr_offset + 64 * r->intra;
            nr_count[r->intra]++;
            for (int i = 0; i < 64; i++) {
                const int v = b[i];
                sum[i] += iabs(v);
                if (v > 0) b[i] = v > off[i] ? v - off[i] : 0;
                else if (v < 0) b[i] = -v > off[i] ? v + off[i] : 0;
            }
        }
        if (r->intra) {
            const int q = (st->h263_aic ? 1 : r->dc_scale) * 8;
            b[0] = (b[0] + q / 2) / q;
        }
        last = trellis ? trellis_quant(st, vlc, inv_aan, b, r->qscale, r->intra, r->lambda2, &ovf, &coded_score[k])
                       : plain_quant(st, b, r->qscale, r->intra, &ovf);
        if (post) {
            const int thr0 = r->chroma ? st->chroma_elim_threshold : st->luma_elim_threshold;
            if (ovf)                                    /* clip the coded range, the intra DC excepted */
                for (int i = r->intra; i <= last; i++) {
                    int16_t *c = &b[st->scantable[i]];
                    *c = *c > st->max_qcoeff ? st->max_qcoeff : *c < st->min_qcoeff ? st->min_qcoeff : *c;
                }
            if (thr0 && !r->intra) {                    /* drop a block of isolated +-1 levels whose run-weighted count is under threshold */
                const int keep_dc = thr0 > 0, thr = iabs(thr0);
                int sc = 0, zeros = 0, big = 0;
                if (last >= keep_dc) {
                    for (int i = 0; i <= last && !big; i++) {
                        const int a = iabs(b[st->scantable[i]]);
                        if (a > 1) big = 1;
                        else if (a == 0) zeros++;
                        else if (!(keep_dc && i == 0)) { sc += zeros == 0 ? 3 : zeros <= 2 ? 2 : zeros <= 23 ? 1 : 0; zeros = 0; }
                    }
                    if (!big && sc < thr) {
                        for (int i = keep_dc; i <= last; i++) b[st->scantable[i]] = 0;
                        last = b[0] ? 0 : -1;
                    }
                }
            }
        }
        last_index[k] = last;
        overflow[k] = ovf;
    }
    return 0;
}
