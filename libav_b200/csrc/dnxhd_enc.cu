// libav_b200/csrc/dnxhd_enc.cu -- the VC-3 / DNxHD encoder (libavcodec/dnxhdenc.c: dnxhd_encode_picture with dnxhd_encode_fast or
// dnxhd_encode_rdo) as one batched call: n frames to n packets, byte-identical to the reference encoder's for the same frames, options and
// rate-control state.
//
// The stages, arithmetic in dnxhd_enc.cuh:
//   qmat    one thread per matrix entry: dnxhd_init_qmat's qmatrix_l / qmatrix_c for qscale 0..qmax.
//   fetch   one thread per 8 x 8 block: dnxhd_get_blocks and the FDCT, once (the reference runs them again for every qscale it tries), and
//           the quantised DC, which does not depend on qscale either.
//   var     one thread per macroblock (fast rate control): dnxhd_mb_var_thread.
//   rank    one thread per macroblock (fast): its place in radix_sort's order.  The values are never negative and passes 2 / 3 are skipped
//           only when they would be identities, so that order is a stable sort by descending value: ties keep macroblock order.
//   rate    one thread per (macroblock, qscale 1..qmax - 1): dnxhd_calc_bits_thread's bits, and in RD mode its SSD.
//   rowsum  one thread per (row, qscale) (fast): the bits of each row, which is all dnxhd_find_qscale reads.
//   search  one CTA per rate-control state: the frames that share it in order, each field through an exact replay of dnxhd_find_qscale +
//           dnxhd_encode_fast or of dnxhd_encode_rdo over the table (32-bit wrap-around, unsigned frame_bits, the row padding and early
//           break), leaving the state as the reference leaves its context.  Its barriers are skipped in a one-thread launch, which is how
//           the host build runs it.
//   layout  one thread per row: slice sizes and each macroblock's bit offset in its slice.
//   header  one thread per coding unit: MSIP offsets, the 640-byte header and the 0x600DC0DE end; the check 640 + offset + 4 <= the
//           coding unit's size.
//   write   one thread per macroblock: its qscale and 8 blocks at its known bit offset, ORed into the zeroed packet.
// Except the search, threads never communicate, so the file also compiles for tests/hostsim/.
#include "common.cuh"
#include "dnxhd_cid.cuh"
#include "dnxhd_enc.cuh"
#include "../../include/avdsp_b200.h"
#include <limits.h>
#include <math.h>
#include <string.h>
#include <vector>

namespace avb {
namespace {

constexpr int DN_FRAMES_PER_LAUNCH = 8;
#ifdef AVB_HOSTSIM
constexpr int DN_SEARCH_THREADS = 1;
#else
constexpr int DN_SEARCH_THREADS = 512;
#endif
struct DnLaunch { DnFrame f[DN_FRAMES_PER_LAUNCH]; int chain[DN_FRAMES_PER_LAUNCH]; };

// ---- kernels ------------------------------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(128) dn_qmat_kernel(const __grid_constant__ DnLaunch L)
{
    const DnFrame &F = L.f[blockIdx.y];
    const unsigned i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= 2u * (F.qmax + 1) * 64) return;
    const int t = (int)(i / ((F.qmax + 1) * 64)), q = (int)(i / 64) % (F.qmax + 1), k = (int)(i & 63);
    const DnTables &T = *F.tab;
    const int j = T.zz[k];
    int v = 0;
    if (q && F.bd == 8) {                                // ff_convert_matrix with weight_matrix[0] = 1, then << 2
        const long long den = (long long)q * (k ? T.weight[t][k] : 1);
        v = F.fdct == 2 ? (int)((1ull << 36) / (unsigned long long)(T.aan[j] * den)) : (int)((1ull << 22) / (unsigned long long)den);
        v = (int)((unsigned)v << 2);
    } else if (q && k) {
        v = (1 << 19) / (q * T.weight[t][k]);
    }
    F.qmat[((size_t)t * (F.qmax + 1) + q) * 64 + j] = v;
}

__global__ void __launch_bounds__(128) dn_fetch_kernel(const __grid_constant__ DnLaunch L)
{
    const DnFrame &F = L.f[blockIdx.y];
    const unsigned i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= (unsigned)F.nf * F.nmb * 8) return;
    const int field = (int)(i / (F.nmb * 8)), mb = (int)(i / 8) % F.nmb, b = (int)(i & 7);
    alignas(16) int16_t s[64];
    dn_fetch_samples(F, field, mb / F.mbw, mb % F.mbw, b, s);
    if (F.rd)
        for (int k = 0; k < 64; k++) F.samp[(size_t)i * 64 + k] = s[k];
    dn_fdct(F, s);
    for (int k = 0; k < 64; k++) F.coef[(size_t)i * 64 + k] = s[k];
    F.dcq[i] = dn_dc(F, s[0]);
}

__global__ void __launch_bounds__(128) dn_var_kernel(const __grid_constant__ DnLaunch L)
{
    const DnFrame &F = L.f[blockIdx.y];
    const unsigned i = blockIdx.x * blockDim.x + threadIdx.x;
    if (F.rd || i >= (unsigned)F.nf * F.nmb) return;
    const int field = (int)(i / F.nmb), mb = (int)(i % F.nmb);
    F.var[i] = dn_mb_var(F, field, mb / F.mbw, mb % F.mbw);
}

__global__ void __launch_bounds__(128) dn_rank_kernel(const __grid_constant__ DnLaunch L)
{
    const DnFrame &F = L.f[blockIdx.y];
    const unsigned i = blockIdx.x * blockDim.x + threadIdx.x;
    if (F.rd || i >= (unsigned)F.nf * F.nmb) return;
    const int field = (int)(i / F.nmb), mb = (int)(i % F.nmb);
    const int32_t *v = F.var + (size_t)field * F.nmb;
    const int me = v[mb];
    int rank = 0;
    for (int j = 0; j < F.nmb; j++) {
        const int o = v[j];
        rank += o > me || (o == me && j < mb);
    }
    F.order[(size_t)field * F.nmb + rank] = mb;
}

__global__ void __launch_bounds__(128) dn_rate_kernel(const __grid_constant__ DnLaunch L)
{
    const DnFrame &F = L.f[blockIdx.y];
    const unsigned i = blockIdx.x * blockDim.x + threadIdx.x;
    const unsigned per_field = (unsigned)(F.qmax - 1) * F.nmb;
    if (i >= per_field * F.nf) return;
    const int field = (int)(i / per_field), r = (int)(i % per_field), q = r / F.nmb + 1, mb = r % F.nmb;
    F.rc[i] = dn_mb_rate(F, field, mb, q);
}

__global__ void __launch_bounds__(128) dn_rowsum_kernel(const __grid_constant__ DnLaunch L)
{
    const DnFrame &F = L.f[blockIdx.y];
    const unsigned i = blockIdx.x * blockDim.x + threadIdx.x;
    if (F.rd || i >= (unsigned)F.nf * (F.qmax - 1) * F.mbh) return;
    const int fq = (int)(i / F.mbh), y = (int)(i % F.mbh);           // fq = field * (qmax - 1) + qscale - 1, as the table's rows
    const DnRc *rc = F.rc + (size_t)fq * F.nmb + (size_t)y * F.mbw;
    int bits = 0;
    for (int x = 0; x < F.mbw; x++) bits += rc[x].bits;
    F.rowbits[i] = bits;
}

// ---- the rate-control search --------------------------------------------------------------------------------------------------------------
struct DnShared {
    int ret, q, lambda, end, done, k;
    long long max_bits;
    int rows[DN_MAX_ROWS];
    long long csum[DN_SEARCH_THREADS], cmax[DN_SEARCH_THREADS];
};
__device__ __forceinline__ void dn_sync()
{
    if (blockDim.x > 1) __syncthreads();            // a one-thread launch (the host build) has nothing to wait for
}
__device__ __forceinline__ const DnRc &dn_rc(const DnFrame &F, int field, int q, int mb)
{
    return F.rc[((size_t)field * (F.qmax - 1) + q - 1) * F.nmb + mb];
}

// dnxhd_find_qscale + dnxhd_encode_fast for one field; returns < 0 when the picture does not fit
__device__ int dn_fast(const DnFrame &F, int field, DnShared &S)
{
    const int tid = (int)threadIdx.x, nt = (int)blockDim.x;
    uint8_t *mbq = F.mbq + (size_t)field * F.nmb;
    int32_t *mbbits = F.mbbits + (size_t)field * F.nmb;
    if (tid == 0) {
        const int32_t *rb = F.rowbits + (size_t)field * (F.qmax - 1) * F.mbh;
        int qscale = (int)F.state->qscale, up_step = 1, down_step = 1, last_higher = 0, last_lower = INT_MAX, ret = 0;
        for (;;) {
            if (qscale < 1 || qscale >= F.qmax) { ret = DN_EINVAL; break; }      // only a state the encoder cannot leave
            F.state->qscale = (unsigned)qscale;
            int bits = 0;
            for (int y = 0; y < F.mbh; y++) {
                bits += rb[(size_t)(qscale - 1) * F.mbh + y];
                bits = (bits + 31) & ~31;                                       // padding
                if ((unsigned)bits > F.frame_bits) break;
            }
            if ((unsigned)bits < F.frame_bits) {
                if (qscale == 1) { ret = 1; break; }
                if (last_higher == qscale - 1) { qscale = last_higher; break; }
                last_lower = min(qscale, last_lower);
                if (last_higher != 0) qscale = (qscale + last_higher) >> 1;
                else qscale -= down_step++;
                if (qscale < 1) qscale = 1;
                up_step = 1;
            } else {
                if (last_lower == qscale + 1) break;
                last_higher = max(qscale, last_higher);
                if (last_lower != INT_MAX) qscale = (qscale + last_lower) >> 1;
                else qscale += up_step++;
                down_step = 1;
                if (qscale >= F.qmax) { ret = DN_EINVAL; break; }
            }
        }
        if (!ret) F.state->qscale = (unsigned)qscale;
        S.ret = ret;
        S.q = (int)F.state->qscale;
        if (ret >= 0) {
            long long max_bits = 0;                      // int in the C code; it cannot wrap: it stays below the sum of all rows' bits
            for (int y = 0; y < F.mbh; y++) max_bits += rb[(size_t)(S.q - 1) * F.mbh + y] + 31;
            S.max_bits = max_bits;
        }
    }
    dn_sync();
    const int ret = S.ret, q = S.q;
    if (ret < 0) return ret;
    for (int mb = tid; mb < F.nmb; mb += nt) { mbq[mb] = (uint8_t)q; mbbits[mb] = dn_rc(F, field, q, mb).bits; }
    if (ret == 1) { dn_sync(); return 0; }
    // the greedy step: the first k macroblocks of the order go to qscale + 1, k where max_bits first drops to frame_bits.  Each thread
    // sums a chunk of the order's deltas and the largest partial sum inside it; one thread then finds the chunk where that happens.
    const int32_t *order = F.order + (size_t)field * F.nmb;
    const int chunk = (F.nmb + nt - 1) / nt, lo = tid * chunk, hi = min(lo + chunk, F.nmb);
    long long sum = 0, best = LLONG_MIN;
    for (int x = lo; x < hi; x++) {
        const int mb = order[x];
        sum += dn_rc(F, field, q, mb).bits - dn_rc(F, field, q + 1, mb).bits;
        if (sum > best) best = sum;
    }
    S.csum[tid] = sum; S.cmax[tid] = best;
    dn_sync();
    if (tid == 0) {
        const long long fb = F.frame_bits;
        long long running = S.max_bits;
        int k = F.nmb;
        for (int c = 0; c < nt && c * chunk < F.nmb; c++) {
            const int clo = c * chunk, chi = min(clo + chunk, F.nmb);
            if (running <= fb) { k = clo; break; }
            if (running - S.cmax[c] <= fb) {
                for (int x = clo; x < chi; x++) {
                    const int mb = order[x];
                    running -= dn_rc(F, field, q, mb).bits - dn_rc(F, field, q + 1, mb).bits;
                    if (running <= fb) { k = x + 1; break; }
                }
                break;
            }
            running -= S.csum[c];
        }
        S.k = k;
    }
    dn_sync();
    for (int x = tid; x < S.k; x += nt) {
        const int mb = order[x];
        mbq[mb] = (uint8_t)(q + 1);
        mbbits[mb] = dn_rc(F, field, q + 1, mb).bits;
    }
    dn_sync();
    return 0;
}

// dnxhd_encode_rdo's lambda search for one field (the table holds every qscale it scores); returns < 0 when the picture does not fit
__device__ int dn_rdo(const DnFrame &F, int field, DnShared &S)
{
    const int tid = (int)threadIdx.x, nt = (int)blockDim.x;
    uint8_t *mbq = F.mbq + (size_t)field * F.nmb;
    int32_t *mbbits = F.mbbits + (size_t)field * F.nmb;
    if (tid == 0) F.state->qscale = (unsigned)(F.qmax - 1);     // the table loop leaves ctx->qscale at qmax - 1 (:783-787)
    int lambda = (int)F.state->lambda, up_step = 2 << DN_LAMBDA_FRAC_BITS, down_step = 2 << DN_LAMBDA_FRAC_BITS;
    int last_lower = INT_MAX, last_higher = 0;
    for (;;) {
        if (tid == 0) {
            S.end = 0;
            if (lambda == last_higher) { lambda++; S.end = 1; }       // need to set final qscales / bits
            S.lambda = lambda;
        }
        dn_sync();
        const unsigned lam = (unsigned)S.lambda;
        for (int mb = tid; mb < F.nmb; mb += nt) {
            unsigned mn = UINT_MAX;
            int qscale = 1;
            for (int q = 1; q < F.qmax; q++) {
                const DnRc e = dn_rc(F, field, q, mb);
                const unsigned score = (unsigned)e.bits * lam + ((unsigned)e.ssd << DN_LAMBDA_FRAC_BITS);
                if (score < mn) { mn = score; qscale = q; }
            }
            mbq[mb] = (uint8_t)qscale;
            mbbits[mb] = dn_rc(F, field, qscale, mb).bits;
        }
        dn_sync();
        for (int y = tid; y < F.mbh; y += nt) {
            int bits = 0;
            for (int x = 0; x < F.mbw; x++) bits += mbbits[y * F.mbw + x];
            S.rows[y] = bits;
        }
        dn_sync();
        if (tid == 0) {
            int bits = 0;
            for (int y = 0; y < F.mbh; y++) {
                bits += S.rows[y];
                bits = (bits + 31) & ~31;                                       // padding
                if ((unsigned)bits > F.frame_bits) break;
            }
            int done = 0, ret = 0;
            if (S.end) {
                done = 1;
                if ((unsigned)bits > F.frame_bits) ret = DN_EINVAL;
            } else if ((unsigned)bits < F.frame_bits) {
                last_lower = min(lambda, last_lower);
                if (last_higher != 0) lambda = (int)((unsigned)lambda + (unsigned)last_higher) >> 1;
                else lambda -= down_step;
                down_step = down_step > INT_MAX / 5 ? INT_MAX : down_step * 5;
                up_step = 1 << DN_LAMBDA_FRAC_BITS;
                lambda = max(1, lambda);
                if (lambda == last_lower) done = 1;
            } else {
                last_higher = max(lambda, last_higher);
                if (last_lower != INT_MAX) lambda = (int)((unsigned)lambda + (unsigned)last_lower) >> 1;
                else if ((long long)lambda + up_step > INT_MAX) { done = 1; ret = DN_EINVAL; }
                else lambda += up_step;
                up_step = up_step > INT_MAX / 5 ? INT_MAX : up_step * 5;
                down_step = 1 << DN_LAMBDA_FRAC_BITS;
            }
            if (done && !ret) F.state->lambda = (unsigned)lambda;       // after the final update, not the lambda the last pass used
            S.done = done; S.ret = ret;
        }
        dn_sync();
        if (S.done) return S.ret;
    }
}

__global__ void __launch_bounds__(DN_SEARCH_THREADS) dn_search_kernel(const __grid_constant__ DnLaunch L)
{
    __shared__ DnShared S;
    for (int k = 0; k < DN_FRAMES_PER_LAUNCH; k++) {
        if (L.chain[k] != (int)blockIdx.x) continue;
        const DnFrame &F = L.f[k];
        if (threadIdx.x == 0)
            for (int field = 0; field < F.nf; field++) F.status[field] = DN_EINVAL;
        int ret = 0;
        for (int field = 0; field < F.nf && ret >= 0; field++) {
            ret = F.rd ? dn_rdo(F, field, S) : dn_fast(F, field, S);
            if (threadIdx.x == 0 && ret >= 0) F.status[field] = 0;
        }
        if (threadIdx.x == 0) {
            F.out_info[0] = ret < 0 ? DN_EINVAL : (int32_t)F.frame_size;
            F.out_info[1] = (int32_t)(F.state->qscale * 118u);        // FF_QP2LAMBDA
        }
        dn_sync();
    }
}

// ---- the packet ---------------------------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(128) dn_layout_kernel(const __grid_constant__ DnLaunch L)
{
    const DnFrame &F = L.f[blockIdx.y];
    const unsigned i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= (unsigned)F.nf * F.mbh) return;
    const int field = (int)(i / F.mbh), y = (int)(i % F.mbh);
    if (F.status[field]) return;
    const size_t m0 = (size_t)field * F.nmb + (size_t)y * F.mbw;
    uint32_t bits = 0;
    for (int x = 0; x < F.mbw; x++) {
        F.mboff[m0 + x] = bits;
        bits += (uint16_t)F.mbbits[m0 + x];                              // ctx->mb_bits is uint16_t
    }
    F.rowbytes[i] = ((bits + 31) & ~31u) >> 3;
}

__device__ inline void dn_be16(uint8_t *p, unsigned v) { p[0] = (uint8_t)(v >> 8); p[1] = (uint8_t)v; }
__device__ inline void dn_be32(uint8_t *p, unsigned v) { dn_be16(p, v >> 16); dn_be16(p + 2, v); }

__global__ void __launch_bounds__(32) dn_header_kernel(const __grid_constant__ DnLaunch L)
{
    const DnFrame &F = L.f[blockIdx.y];
    const int field = (int)threadIdx.x;
    if (field >= F.nf || F.status[field]) return;
    uint8_t *buf = F.out + (size_t)field * F.cu_size;
    const uint32_t *rows = F.rowbytes + (size_t)field * F.mbh;
    uint32_t offset = 0;
    for (int y = 0; y < F.mbh; y++) {
        F.sliceoff[(size_t)field * F.mbh + y] = offset;
        dn_be32(buf + 0x170 + 4 * y, offset);                                // MSIP
        offset += rows[y];
    }
    if (640ull + offset + 4 > F.cu_size) {                                   // the reference asserts; here the frame fails
        F.status[field] = DN_EINVAL;
        F.out_info[0] = DN_EINVAL;
        return;
    }
    const int cur_field = F.first_field ^ field;
    buf[0] = 0x00; buf[1] = 0x00; buf[2] = 0x02; buf[3] = 0x80; buf[4] = 0x01;
    buf[5] = F.il ? (uint8_t)(cur_field + 2) : 0x01;
    buf[6] = 0x80;                                                           // crc flag off
    buf[7] = 0xa0;
    dn_be16(buf + 0x18, (unsigned)F.height >> F.il);                         // ALPF
    dn_be16(buf + 0x1a, (unsigned)F.width);                                  // SPL
    dn_be16(buf + 0x1d, (unsigned)F.height >> F.il);                         // NAL
    buf[0x21] = F.bd == 10 ? 0x58 : 0x38;
    buf[0x22] = (uint8_t)(0x88 + (F.il << 2));
    dn_be32(buf + 0x28, (unsigned)F.cid);
    buf[0x2c] = F.il ? 0 : 0x80;
    buf[0x5f] = 0x01;                                                        // UDL
    buf[0x167] = 0x02;
    dn_be16(buf + 0x16a, (unsigned)F.mbh * 4 + 4);                           // MSIPS
    buf[0x16d] = (uint8_t)F.mbh;                                             // Ns
    buf[0x16f] = 0x10;
    dn_be32(buf + F.cu_size - 4, 0x600DC0DEu);                               // EOF
}

__global__ void __launch_bounds__(128) dn_write_kernel(const __grid_constant__ DnLaunch L)
{
    const DnFrame &F = L.f[blockIdx.y];
    const unsigned i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= (unsigned)F.nf * F.nmb) return;
    const int field = (int)(i / F.nmb), mb = (int)(i % F.nmb);
    if (F.status[field]) return;
    const size_t slice = 640 + F.sliceoff[(size_t)field * F.mbh + mb / F.mbw];
    dn_write_mb(F, field, mb, reinterpret_cast<uint32_t *>(F.out + (size_t)field * F.cu_size), slice * 8 + F.mboff[i]);
}

// ---- host side ------------------------------------------------------------------------------------------------------------------------------
int dn_refuse(const char *msg) { set_error_msg("ff_dnxhd_encode_frames_cuda", msg); return -1; }

// dnxhd_init_vlc and the fixed tables on the host; -1 (with a message) for an entry the reference's asserts would reject
int dn_build_tables(const FFDnxhdCidEntry &e, DnTables &T)
{
    memset(&T, 0, sizeof(T));
    const int ml = 1 << (e.bit_depth + 2);
    T.max_level = ml;
    for (int level = -ml; level < ml; level++) {
        for (int run = 0; run < 2; run++) {
            const int index = 2 * ml + level * 2 + run;
            const int sign = level < 0 ? -1 : 0;
            int alevel = level < 0 ? -level : level, offset = 0, j;
            if (alevel > 64) { offset = (alevel - 1) >> 6; alevel -= offset << 6; }
            for (j = 0; j < 257; j++) {
                if (e.ac_level[j] == alevel && (!offset || e.ac_index_flag[j]) && (!run || e.ac_run_flag[j])) {
                    if (alevel) { T.vlc_codes[index] = ((uint32_t)e.ac_codes[j] << 1) | (sign & 1); T.vlc_bits[index] = e.ac_bits[j] + 1; }
                    else { T.vlc_codes[index] = e.ac_codes[j]; T.vlc_bits[index] = e.ac_bits[j]; }
                    break;
                }
            }
            if (alevel && j == 257) return dn_refuse("the CID entry has no code for a level (dnxhd_init_vlc would assert)");
            if (offset) { T.vlc_codes[index] = (T.vlc_codes[index] << e.index_bits) | offset; T.vlc_bits[index] += e.index_bits; }
        }
    }
    bool seen[64] = {};
    for (int i = 0; i < 62; i++) {
        const int run = e.run[i];
        if (run < 1 || run > 62 || seen[run])
            return dn_refuse("the CID entry's run table has a run of 0, a run past 62 or a run listed twice");
        seen[run] = true;
        T.run_codes[run] = e.run_codes[i];
        T.run_bits[run] = e.run_bits[i];
    }
    for (int i = 0; i < e.bit_depth + 4; i++) { T.dc_codes[i] = e.dc_codes[i]; T.dc_bits[i] = e.dc_bits[i]; }
    memcpy(T.weight[0], e.luma_weight, 64);
    memcpy(T.weight[1], e.chroma_weight, 64);
    int k = 0;                                                            // ff_zigzag_direct: the anti-diagonals, alternating direction
    for (int s = 0; s < 15; s++) {
        const int r0 = s < 8 ? 0 : s - 7, r1 = s < 8 ? s : 7;
        for (int n = 0; n <= r1 - r0; n++) {
            const int r = s & 1 ? r0 + n : r1 - n;
            T.zz[k++] = (uint8_t)(8 * r + s - r);
        }
    }
    const double pi = 3.14159265358979323846;                              // ff_aanscales: 16384 a(u) a(v), a(0) = 1, a(k) = sqrt(2) cos(k pi / 16)
    for (int i = 0; i < 64; i++) {
        const int u = i >> 3, v = i & 7;
        const double au = u ? sqrt(2.0) * cos(u * pi / 16) : 1.0, av = v ? sqrt(2.0) * cos(v * pi / 16) : 1.0;
        T.aan[i] = (uint16_t)floor(16384.0 * au * av + 0.5);
    }
    return 0;
}

size_t dn_align(size_t v) { return (v + 255) & ~(size_t)255; }

// the frame's workspace arrays in order: {bytes} for each, sized from the derived geometry
struct DnSizes { size_t coef, samp, dcq, qmat, rc, rowbits, var, order, mbq, mbbits, mboff, rows, status; };
DnSizes dn_sizes(const DnFrame &F)
{
    const size_t nb = (size_t)F.nf * F.nmb, Q = (size_t)F.qmax - 1, fast = !F.rd;
    return DnSizes{ nb * 8 * 128, F.rd ? nb * 8 * 128 : 0, nb * 16, 2 * ((size_t)F.qmax + 1) * 256, Q * nb * sizeof(DnRc),
                    fast * Q * F.nf * F.mbh * 4, fast * nb * 4, fast * nb * 4, nb, nb * 4, nb * 4, (size_t)F.nf * F.mbh * 4, 16 };
}
size_t dn_bytes(const DnFrame &F)
{
    const DnSizes z = dn_sizes(F);
    return dn_align(z.coef) + dn_align(z.samp) + dn_align(z.dcq) + dn_align(z.qmat) + dn_align(z.rc) + dn_align(z.rowbits) + dn_align(z.var) +
           dn_align(z.order) + dn_align(z.mbq) + dn_align(z.mbbits) + dn_align(z.mboff) + 2 * dn_align(z.rows) + dn_align(z.status);
}

// the checks and encode_init's derivations for one frame; fills F's geometry (not its tables or workspace pointers)
int dn_frame(const FFDnxhdEncodeWork &w, DnFrame &F)
{
    const FFDnxhdCidEntry *e = w.cid_table;
    if (!e) return dn_refuse("NULL cid_table");
    if (e->bit_depth != 8 && e->bit_depth != 10) return dn_refuse("the CID entry's bit depth must be 8 or 10");
    if (e->interlaced != 0 && e->interlaced != 1) return dn_refuse("the CID entry's interlaced must be 0 or 1");
    if (w.interlaced < 0 || w.interlaced > 2 || (w.interlaced != 0) != (e->interlaced != 0))
        return dn_refuse("interlaced must be 0 for a progressive CID and 1 (top field first) or 2 (bottom field first) for an interlaced one");
    if (!e->width || !e->height || e->width > 4096 || ((e->height + 15) / 16) / (e->interlaced ? 2 : 1) > DN_MAX_ROWS)
        return dn_refuse("the CID entry's size is outside what DNxHD codes (up to 68 macroblock rows per coding unit)");
    if (!e->luma_weight || !e->chroma_weight || !e->dc_codes || !e->dc_bits || !e->ac_codes || !e->ac_bits || !e->ac_level ||
        !e->ac_run_flag || !e->ac_index_flag || !e->run_codes || !e->run_bits || !e->run)
        return dn_refuse("the CID entry has a NULL table");
    if (w.qmax < 2 || w.qmax > DN_QMAX) return dn_refuse("qmax must be 2..69");
    if (w.nitris_compat != 0 && w.nitris_compat != 1) return dn_refuse("nitris_compat must be 0 or 1");
    const int nf = e->interlaced ? 2 : 1;
    const unsigned min_padding = w.nitris_compat ? 1600 : 0;
    if ((e->coding_unit_size & 3) || e->coding_unit_size < 644 + min_padding || e->frame_size < (unsigned)nf * e->coding_unit_size)
        return dn_refuse("the CID entry's coding unit must be a multiple of 4 bytes above 644 + min_padding and fit its frame size");
    const int bpp = e->bit_depth == 8 ? 1 : 2;
    for (int p = 0; p < 3; p++) {
        if (!w.data[p] || (bpp == 2 && ((uintptr_t)w.data[p] & 1))) return dn_refuse("NULL or odd plane pointer");
        if (w.linesize[p] <= 0 || (bpp == 2 && (w.linesize[p] & 1))) return dn_refuse("linesize must be positive, and even at 10 bit");
        if ((long)w.linesize[p] < (long)bpp * (p ? e->width / 2 : e->width)) return dn_refuse("linesize narrower than the plane");
    }
    if (!w.state || ((uintptr_t)w.state & 3)) return dn_refuse("NULL or misaligned state");
    if (!w.out_info || ((uintptr_t)w.out_info & 3)) return dn_refuse("NULL or misaligned out_info");
    if (!w.out || ((uintptr_t)w.out & 3)) return dn_refuse("NULL or misaligned (not 4-byte) out");
    if (w.out_capacity < e->frame_size) return dn_refuse("out_capacity is smaller than the CID's frame_size");
    memset(&F, 0, sizeof(F));
    for (int p = 0; p < 3; p++) { F.data[p] = w.data[p]; F.ls[p] = w.linesize[p]; }
    F.cid = e->cid; F.width = (int)e->width; F.height = (int)e->height; F.bd = e->bit_depth;
    F.il = e->interlaced; F.nf = nf; F.first_field = w.interlaced == 2;
    F.fdct = w.dct_algo == 1 ? 2 : w.dct_algo == 6 ? 6 : 0;                 // FF_DCT_FASTINT, FF_DCT_FAAN, else islow
    F.rd = w.mb_decision == 2;                                              // FF_MB_DECISION_RD
    F.qmax = w.qmax;
    F.mbw = (F.width + 15) / 16;
    F.mbh = (F.height + 15) / 16 / nf;
    F.nmb = F.mbw * F.mbh;
    F.frame_bits = (e->coding_unit_size - 640 - 4 - min_padding) * 8;
    F.frame_size = e->frame_size; F.cu_size = e->coding_unit_size;
    F.state = w.state; F.out = w.out; F.out_info = w.out_info;
    return 0;
}

void dn_place(DnFrame &F, uint8_t *&ws)
{
    const DnSizes z = dn_sizes(F);
    auto take = [&](size_t n) { uint8_t *p = n ? ws : nullptr; ws += dn_align(n); return p; };
    F.coef = reinterpret_cast<int16_t *>(take(z.coef));
    F.samp = reinterpret_cast<int16_t *>(take(z.samp));
    F.dcq = reinterpret_cast<int16_t *>(take(z.dcq));
    F.qmat = reinterpret_cast<int32_t *>(take(z.qmat));
    F.rc = reinterpret_cast<DnRc *>(take(z.rc));
    F.rowbits = reinterpret_cast<int32_t *>(take(z.rowbits));
    F.var = reinterpret_cast<int32_t *>(take(z.var));
    F.order = reinterpret_cast<int32_t *>(take(z.order));
    F.mbq = take(z.mbq);
    F.mbbits = reinterpret_cast<int32_t *>(take(z.mbbits));
    F.mboff = reinterpret_cast<uint32_t *>(take(z.mboff));
    F.rowbytes = reinterpret_cast<uint32_t *>(take(z.rows));
    F.sliceoff = reinterpret_cast<uint32_t *>(take(z.rows));
    F.status = reinterpret_cast<int32_t *>(take(z.status));
}

unsigned dn_blocks(size_t threads) { return (unsigned)((threads + 127) / 128); }
size_t dn_max(size_t a, size_t b) { return a > b ? a : b; }

int dn_launch(const DnLaunch &L, int m, int nchains, cudaStream_t st)
{
    size_t nq = 0, nblk = 0, nmb = 0, nrate = 0, nrowq = 0, nrows = 0;
    for (int k = 0; k < m; k++) {
        const DnFrame &F = L.f[k];
        nq = dn_max(nq, 2 * ((size_t)F.qmax + 1) * 64);
        nblk = dn_max(nblk, (size_t)F.nf * F.nmb * 8);
        nmb = dn_max(nmb, (size_t)F.nf * F.nmb);
        nrate = dn_max(nrate, (size_t)F.nf * (F.qmax - 1) * F.nmb);
        nrowq = dn_max(nrowq, F.rd ? 0 : (size_t)F.nf * (F.qmax - 1) * F.mbh);
        nrows = dn_max(nrows, (size_t)F.nf * F.mbh);
    }
    const char *where = "ff_dnxhd_encode_frames_cuda";
    for (int k = 0; k < m; k++)                                             // the padding between slices and after the last is zero
        if (cudaMemsetAsync(L.f[k].out, 0, L.f[k].frame_size, st) != cudaSuccess) { set_error(where, cudaGetLastError()); return -1; }
    AVB_LAUNCH(dn_qmat_kernel, dim3(dn_blocks(nq), m), dim3(128), 0, st)(L);
    if (check_launch(where)) return -1;
    AVB_LAUNCH(dn_fetch_kernel, dim3(dn_blocks(nblk), m), dim3(128), 0, st)(L);
    if (check_launch(where)) return -1;
    if (nrowq) {
        AVB_LAUNCH(dn_var_kernel, dim3(dn_blocks(nmb), m), dim3(128), 0, st)(L);
        if (check_launch(where)) return -1;
        AVB_LAUNCH(dn_rank_kernel, dim3(dn_blocks(nmb), m), dim3(128), 0, st)(L);
        if (check_launch(where)) return -1;
    }
    AVB_LAUNCH(dn_rate_kernel, dim3(dn_blocks(nrate), m), dim3(128), 0, st)(L);
    if (check_launch(where)) return -1;
    if (nrowq) {
        AVB_LAUNCH(dn_rowsum_kernel, dim3(dn_blocks(nrowq), m), dim3(128), 0, st)(L);
        if (check_launch(where)) return -1;
    }
    AVB_LAUNCH(dn_search_kernel, dim3(nchains), dim3(DN_SEARCH_THREADS), 0, st)(L);
    if (check_launch(where)) return -1;
    AVB_LAUNCH(dn_layout_kernel, dim3(dn_blocks(nrows), m), dim3(128), 0, st)(L);
    if (check_launch(where)) return -1;
    AVB_LAUNCH(dn_header_kernel, dim3(1, m), dim3(32), 0, st)(L);
    if (check_launch(where)) return -1;
    AVB_LAUNCH(dn_write_kernel, dim3(dn_blocks(nmb), m), dim3(128), 0, st)(L);
    return check_launch(where);
}

size_t dn_workspace(const FFDnxhdEncodeWork *frames, int n)
{
    if (!frames || n < 1) return 0;
    size_t total = 0;
    for (int k = 0; k < n; k++) {
        DnFrame F;
        if (dn_frame(frames[k], F)) return 0;
        total += dn_bytes(F);
    }
    return total;
}

}  // namespace
}  // namespace avb

using namespace avb;

extern "C" {

size_t ff_dnxhd_encode_workspace_cuda(const FFDnxhdEncodeWork *frames, int n)
{
    return dn_workspace(frames, n);
}

int ff_dnxhd_encode_frames_cuda(const FFDnxhdEncodeWork *frames, int n, void *workspace, size_t workspace_bytes, void *stream)
{
    avb::enter();
    if (n == 0) return 0;
    if (!frames || n < 0) return dn_refuse("NULL frames or a negative count");
    size_t need = 0;
    std::vector<const DnTables *> tabs(n);
    for (int k = 0; k < n; k++) {                         // every frame is checked before anything is launched
        DnFrame F;
        if (dn_frame(frames[k], F)) return -1;
        need += dn_bytes(F);
    }
    if (!workspace || workspace_bytes < need) return dn_refuse("workspace missing or smaller than ff_dnxhd_encode_workspace_cuda returns");
    for (int k = 0; k < n; k++)
        if (!(tabs[k] = dn_tables_cached<DnTables>(frames[k].cid_table, dn_build_tables, "ff_dnxhd_encode_frames_cuda"))) return -1;
    uint8_t *ws = (uint8_t *)workspace;
    for (int g0 = 0; g0 < n; g0 += DN_FRAMES_PER_LAUNCH) {
        const int m = n - g0 < DN_FRAMES_PER_LAUNCH ? n - g0 : DN_FRAMES_PER_LAUNCH;
        DnLaunch L;
        memset(&L, 0, sizeof(L));
        int nchains = 0;
        for (int k = 0; k < DN_FRAMES_PER_LAUNCH; k++) L.chain[k] = -1;
        for (int k = 0; k < m; k++) {
            dn_frame(frames[g0 + k], L.f[k]);
            L.f[k].tab = tabs[g0 + k];
            dn_place(L.f[k], ws);
            for (int j = 0; j < k && L.chain[k] < 0; j++)
                if (L.f[j].state == L.f[k].state) L.chain[k] = L.chain[j];
            if (L.chain[k] < 0) L.chain[k] = nchains++;
        }
        if (dn_launch(L, m, nchains, (cudaStream_t)stream)) return -1;
    }
    return 0;
}

}  // extern "C"
