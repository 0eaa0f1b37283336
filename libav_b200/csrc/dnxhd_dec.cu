// libav_b200/csrc/dnxhd_dec.cu -- the VC-3 / DNxHD decoder (libavcodec/dnxhddec.c: dnxhd_decode_frame) as one batched call: n packets to n
// frames, every sample the reference decoder writes written with its value.
//
// Every macroblock row of a coding unit starts at its own byte offset (mb_scan_index) with last_dc reset, so rows are independent.  Two
// stages, arithmetic in dnxhd_dec.cuh:
//   entropy  one thread per (coding unit, row): the macroblocks' qscale, interlaced_mb and dequantised blocks into the workspace.  A CTA
//            is one warp holding rows of one packet and stages that packet's lookup tables in shared memory.  A warp has `lanes` active
//            threads, the fewest that keep all of a launch's CTAs resident at once (dd_lanes).  A call of up to 64 packets is one launch.
//   put      one thread per 8 x 8 block: ff_simple_idct_put_8 / _10 at the block's place.  The second field is put after the first,
//            because with interlaced_mb or equal cur_field the two write the same lines and the reference's order decides.
// The table staging's barrier is skipped in a one-thread CTA, which is how the host build (tests/hostsim/) runs the entropy stage.
#include "common.cuh"
#include "dnxhd_cid.cuh"
#include "dnxhd_dec.cuh"
#include "../../include/avdsp_b200.h"
#include <string.h>
#include <vector>

namespace avb {
namespace {

constexpr int DD_FRAMES_PER_LAUNCH = 64;        // a call of up to 64 packets is one launch per stage (kernel parameters of 8.7 KB, sm_70+)
#ifdef AVB_HOSTSIM
constexpr int DD_ENTROPY_THREADS = 1;
#else
constexpr int DD_ENTROPY_THREADS = 32;
#endif
constexpr int DD_INVALIDDATA = -0x3ebbb1b7;                  // AVERROR_INVALIDDATA
constexpr int DD_ENOSYS = -38, DD_EINVAL = -22;
struct DdLaunch { DdFrame f[DD_FRAMES_PER_LAUNCH]; int lanes; };
static_assert(sizeof(DdLaunch) <= 32764, "kernel parameters");

// ---- kernels ------------------------------------------------------------------------------------------------------------------------------
// A CTA is one warp (one thread in the host build) and takes `lanes` consecutive rows of one packet, one per lane.
__global__ void __launch_bounds__(DD_ENTROPY_THREADS) dd_entropy_kernel(const __grid_constant__ DdLaunch L)
{
    __shared__ DdTables S;
    const DdFrame &F = L.f[blockIdx.y];
    const int lane = (int)threadIdx.x, first = (int)blockIdx.x * L.lanes, t = first + lane;
    if (first >= F.rows) return;                                              // the whole CTA: no barrier is pending
    const uint4 *src = reinterpret_cast<const uint4 *>(F.tab);
    uint4 *dst = reinterpret_cast<uint4 *>(&S);
    for (int k = (int)threadIdx.x; k < (int)(sizeof(DdTables) / 16); k += (int)blockDim.x) dst[k] = src[k];
    if (blockDim.x > 1) __syncthreads();
    if (lane >= L.lanes || t >= F.rows) return;
    dd_row(F, S, t);
}

__global__ void __launch_bounds__(128) dd_put_kernel(const __grid_constant__ DdLaunch L, int unit)
{
    const DdFrame &F = L.f[blockIdx.y];
    if (unit >= F.nu) return;
    const int nb = F.is444 ? 12 : 8, per_row = F.mbw * nb;
    const unsigned i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= (unsigned)(F.u[unit].mbh * per_row)) return;
    const int t = (unit ? F.u[0].mbh : 0) + (int)(i / per_row), r = (int)(i % per_row);
    dd_put_block(F, t, r / nb, r % nb);
}

// ---- host side ------------------------------------------------------------------------------------------------------------------------------
int dd_refuse(const char *where, const char *msg) { set_error_msg(where, msg); return -1; }

// one code table of an entry (n codes with their lengths; length 0: no code, as init_vlc skips it) into a two-level lookup at t[0..cap)
// with the given leaf payloads; -1 unless the codes form a complete prefix code of at most 16 bits that fits
int dd_build_vlc(const uint16_t *codes16, const uint8_t *codes8, const uint8_t *bits, int n, const uint16_t *payload, uint16_t *t, int cap)
{
    std::vector<uint32_t> filled(cap, 0);
    int used = 1 << DD_VLC_BITS;
    for (int s = 0; s < n; s++) {
        const int len = bits[s];
        if (!len) continue;
        const uint32_t code = codes16 ? codes16[s] : codes8[s];
        if (len > 16 || code >> len) return -1;
        if (len <= DD_VLC_BITS) {
            const uint32_t lo = code << (DD_VLC_BITS - len), hi = lo + (1u << (DD_VLC_BITS - len));
            for (uint32_t k = lo; k < hi; k++) {
                if (filled[k]) return -1;
                filled[k] = 1; t[k] = (uint16_t)(payload[s] << 5 | len);
            }
            continue;
        }
        const uint32_t pre = code >> (len - DD_VLC_BITS);
        if (filled[pre] && !(t[pre] & 0x8000u)) return -1;
        if (!filled[pre]) {
            if (used + (1 << DD_SUB_BITS) > cap) return -1;
            filled[pre] = 1; t[pre] = (uint16_t)(0x8000u | used);
            used += 1 << DD_SUB_BITS;
        }
        const uint32_t base = t[pre] & 0x7fffu, rest = code & ((1u << (len - DD_VLC_BITS)) - 1);
        const uint32_t lo = rest << (16 - len), hi = lo + (1u << (16 - len));
        for (uint32_t k = lo; k < hi; k++) {
            if (filled[base + k]) return -1;
            filled[base + k] = 1; t[base + k] = (uint16_t)(payload[s] << 5 | len);
        }
    }
    for (int k = 0; k < used; k++)                                            // complete: every pattern reaches a code
        if (!filled[k]) return -1;
    return 0;
}

int dd_build_tables(const FFDnxhdCidEntry &e, DdTables &T, const char *where)
{
    memset(&T, 0, sizeof(T));
    uint16_t pay[257];
    for (int s = 0; s < 257; s++) pay[s] = (uint16_t)(e.ac_level[s] | (e.ac_index_flag[s] ? 0x100 : 0) | (e.ac_run_flag[s] ? 0x200 : 0));
    if (dd_build_vlc(e.ac_codes, nullptr, e.ac_bits, 257, pay, T.ac, DD_AC_N))
        return dd_refuse(where, "the CID entry's AC codes are not a complete prefix code of at most 16 bits, or need more than 24 second-level tables");
    for (int s = 0; s < 62; s++) pay[s] = e.run[s];
    if (dd_build_vlc(e.run_codes, nullptr, e.run_bits, 62, pay, T.run, DD_RUN_N))
        return dd_refuse(where, "the CID entry's run codes are not a complete prefix code of at most 16 bits, or need more than 32 second-level tables");
    bool seen[128] = {};
    for (int s = 0; s < e.bit_depth + 4; s++) {
        const int len = e.dc_bits[s], code = e.dc_codes[s];
        if (!len) continue;
        if (len > 7 || code >> len) return dd_refuse(where, "the CID entry has a DC code longer than 7 bits or wider than its length");
        for (int k = code << (7 - len); k < (code + 1) << (7 - len); k++) {
            if (seen[k]) return dd_refuse(where, "the CID entry's DC codes are not a prefix code");
            seen[k] = true; T.dc[k] = (uint8_t)(s << 3 | len);
        }
    }
    for (int k = 0; k < 128; k++)
        if (!seen[k]) return dd_refuse(where, "the CID entry's DC codes are not a complete prefix code");
    memcpy(T.weight[0], e.luma_weight, 64);
    memcpy(T.weight[1], e.chroma_weight, 64);
    int k = 0;                                                                // ff_zigzag_direct: the anti-diagonals, alternating direction
    for (int s = 0; s < 15; s++) {
        const int r0 = s < 8 ? 0 : s - 7, r1 = s < 8 ? s : 7;
        for (int n = 0; n <= r1 - r0; n++) {
            const int r = s & 1 ? r0 + n : r1 - n;
            T.zz[k++] = (uint8_t)(8 * r + s - r);
        }
    }
    return 0;
}

// av_reduce(num, den, max) for the non-negative values the header gives: the best approximation with both terms at most max, from the
// continued fraction's convergents and the last semiconvergent
void dd_reduce(int64_t num, int64_t den, int64_t max, int *out_num, int *out_den)
{
    int64_t a = num, b = den;
    while (b) { const int64_t r = a % b; a = b; b = r; }
    if (a) { num /= a; den /= a; }
    int64_t p0 = 0, q0 = 1, p1 = 1, q1 = 0;
    if (num <= max && den <= max) { p1 = num; q1 = den; den = 0; }
    while (den) {
        int64_t x = num / den;
        const int64_t next = num - den * x, p2 = x * p1 + p0, q2 = x * q1 + q0;
        if (p2 > max || q2 > max) {
            if (p1) x = (max - p0) / p1;
            if (q1) x = x < (max - q0) / q1 ? x : (max - q0) / q1;
            if (den * (2 * x * q1 + q0) > num * q1) { p1 = x * p1 + p0; q1 = x * q1 + q0; }
            break;
        }
        p0 = p1; q0 = q1; p1 = p2; q1 = q2;
        num = den; den = next;
    }
    *out_num = (int)p1; *out_den = (int)q1;
}

// what dnxhd_decode_header derives for one coding unit
struct DdHeader { int cid, bd, is444, il, cur_field, mbaff, width, height, mbh, sar_num, sar_den; const FFDnxhdCidEntry *e; };

// dnxhd_decode_header for the unit at buf (buf_size bytes to the packet's end); frame_il: whether an earlier unit made the frame interlaced
int dd_header(const uint8_t *buf, long buf_size, int frame_il, const FFDnxhdCidEntry *cids, int n_cids, DdHeader &h, const char *where)
{
    static const uint8_t prefix[5] = { 0x00, 0x00, 0x02, 0x80, 0x01 }, prefix444[5] = { 0x00, 0x00, 0x02, 0x80, 0x02 };
    memset(&h, 0, sizeof(h));
    h.sar_num = 0; h.sar_den = 1;
    if (buf_size < 0x280) return DD_INVALIDDATA;
    if (memcmp(buf, prefix, 5) && memcmp(buf, prefix444, 5)) return DD_INVALIDDATA;
    h.il = frame_il;
    if (buf[5] & 2) { h.il = 1; h.cur_field = buf[5] & 1; }
    h.mbaff = (buf[6] & 32) != 0;
    h.height = buf[0x18] << 8 | buf[0x19];
    h.width = buf[0x1a] << 8 | buf[0x1b];
    if (buf[0x21] == 0x58) { h.bd = 10; h.is444 = buf[4] == 2; }
    else if (buf[0x21] == 0x38) h.bd = 8;
    else return DD_INVALIDDATA;
    h.cid = (int)dd_be32(buf + 0x28);
    if (!h.cid) return dd_refuse(where, "CID 0 (a fresh reference context takes it for its cached CID and never sets its table)");
    for (int k = 0; k < n_cids && !h.e; k++)
        if (cids[k].cid == h.cid) h.e = &cids[k];
    if (!h.e) return DD_ENOSYS;
    if (h.width != (int)h.e->width) {
        dd_reduce(h.width, h.e->width, 255, &h.sar_num, &h.sar_den);
        h.width = (int)h.e->width;
    }
    if ((unsigned long)buf_size < h.e->coding_unit_size) return DD_INVALIDDATA;
    h.mbh = buf[0x16d];
    if ((h.height + 15) >> 4 == h.mbh && h.il) h.height <<= 1;
    if (h.mbh > DD_MAX_ROWS || (h.mbh << h.il) > (h.height + 15) >> 4) return DD_INVALIDDATA;
    for (int i = 0; i < h.mbh; i++) {
        const uint32_t idx = dd_be32(buf + 0x170 + 4 * i);
        if (idx > 0xffffffffu - 0x280) return dd_refuse(where, "a scan index within 0x280 of 2^32 (the reference's bound check wraps)");
        if ((unsigned long)buf_size < idx + 0x280ul) return DD_INVALIDDATA;
    }
    if (h.bd != h.e->bit_depth) return dd_refuse(where, "the header's bit depth is not its CID entry's bit_depth");
    return 0;
}

// the probe, and the units of the packet for the kernels (u, nu); ff_set_dimensions's av_image_check_size after each header
int dd_probe(const uint8_t *pkt, int size, const FFDnxhdCidEntry *cids, int n_cids, FFDnxhdFrameInfo &info, DdUnit *u, int &nu,
             const DdTables **tab, const char *where)
{
    memset(&info, 0, sizeof(info));
    if (!pkt || size < 0) return dd_refuse(where, "NULL packet or a negative size");
    if (!cids || n_cids < 0) return dd_refuse(where, "NULL CID table or a negative count");
    DdHeader h0, h1;
    int ret = dd_header(pkt, size, 0, cids, n_cids, h0, where);
    if (ret) return ret;
    auto check_size = [](int w, int h) { return w > 0 && h > 0 && (uint64_t)(w + 128) * (uint64_t)(h + 128) < (uint64_t)(0x7fffffff / 8); };
    if (!check_size(h0.width, h0.height)) return DD_EINVAL;
    nu = 1;
    u[0] = DdUnit{ 0, h0.mbh, h0.mbaff, h0.cur_field };
    int tff = h0.il ? 1 ^ h0.cur_field : 0, mbh = h0.mbh;
    if (h0.il) {
        const uint32_t cu = h0.e->coding_unit_size;
        ret = dd_header(pkt + cu, (long)size - (long)cu, 1, cids, n_cids, h1, where);
        if (ret) return ret;
        if (!(pkt[cu + 5] & 2) || h1.cid != h0.cid || h1.bd != h0.bd || h1.is444 != h0.is444 || h1.width != h0.width || h1.height != h0.height)
            return dd_refuse(where, "the second coding unit is not an interlaced field header with the first unit's CID, bit depth, chroma "
                                    "format and size");
        nu = 2;
        u[1] = DdUnit{ cu, h1.mbh, h1.mbaff, h1.cur_field };
        tff = h1.cur_field;
        mbh = mbh > h1.mbh ? mbh : h1.mbh;
    }
    auto build = [where](const FFDnxhdCidEntry &e, DdTables &T) { return dd_build_tables(e, T, where); };
    if (tab) {
        if (!(*tab = dn_tables_cached<DdTables>(h0.e, build, where))) return -1;
    } else {                                                                  // the entry's checks without the device copy
        std::vector<uint8_t> host(sizeof(DdTables));
        if (build(*h0.e, *reinterpret_cast<DdTables *>(host.data()))) return -1;
    }
    info.cid = h0.cid;
    info.width = h0.width;
    info.height = h0.height;
    info.pix_fmt = h0.bd == 8 ? FF_DNXHD_PIX_FMT_YUV422P : h0.is444 ? FF_DNXHD_PIX_FMT_YUV444P10 : FF_DNXHD_PIX_FMT_YUV422P10;
    info.interlaced_frame = h0.il;
    info.top_field_first = tff;
    info.sar_num = h0.sar_num; info.sar_den = h0.sar_den;
    info.lines = (mbh * 16) << h0.il;
    return 0;
}

// the checks of one packet and its planes; fills F's geometry (not its workspace pointers)
int dd_frame(const FFDnxhdDecodeWork &w, const FFDnxhdCidEntry *cids, int n_cids, DdFrame &F, bool tables)
{
    const char *where = "ff_dnxhd_decode_frames_cuda";
    memset(&F, 0, sizeof(F));
    FFDnxhdFrameInfo info;
    int nu = 0;
    const int ret = dd_probe(w.pkt_host, w.size, cids, n_cids, info, F.u, nu, tables ? &F.tab : nullptr, where);
    if (ret > 0 || ret < -1) return dd_refuse(where, "a packet the decoder refuses (ff_dnxhd_probe_cuda returns its AVERROR)");
    if (ret) return -1;
    if (!w.pkt) return dd_refuse(where, "NULL device packet");
    const int bd10 = info.pix_fmt != FF_DNXHD_PIX_FMT_YUV422P, is444 = info.pix_fmt == FF_DNXHD_PIX_FMT_YUV444P10;
    for (int p = 0; p < 3; p++) {
        const long width = (long)(p && !is444 ? info.width / 2 : info.width) << bd10;
        if (p && w.gray) continue;
        if (!w.data[p] || (bd10 && ((uintptr_t)w.data[p] & 1))) return dd_refuse(where, "NULL or odd plane pointer");
        if (w.linesize[p] <= 0 || (bd10 && (w.linesize[p] & 1)) || w.linesize[p] < width)
            return dd_refuse(where, "linesize must be positive, even at 10 bit and at least the plane's width in bytes");
        if (w.lines[p] < info.lines) return dd_refuse(where, "a plane holds fewer lines than the frame needs");
    }
    if (!w.gray && w.linesize[1] != w.linesize[2]) return dd_refuse(where, "the U and V linesizes differ");
    F.pkt = w.pkt; F.size = (uint32_t)w.size;
    for (int p = 0; p < 3; p++) { F.data[p] = w.data[p]; F.ls[p] = w.linesize[p]; }
    F.mbw = (int)(info.width >> 4);
    F.nu = nu;
    F.rows = F.u[0].mbh + (nu > 1 ? F.u[1].mbh : 0);
    F.bd10 = bd10; F.is444 = is444; F.il = info.interlaced_frame; F.gray = w.gray != 0;
    return 0;
}

size_t dd_align(size_t v) { return (v + 255) & ~(size_t)255; }
size_t dd_coef_bytes(const DdFrame &F) { return (size_t)F.rows * F.mbw * (F.is444 ? 12 : 8) * 128; }
size_t dd_bytes(const DdFrame &F) { return dd_align(dd_coef_bytes(F)) + dd_align((size_t)F.rows * F.mbw); }

// active lanes per entropy warp for a launch of `rows` rows: the fewest that still fit every CTA on the device at once (resident CTAs per
// SM, which the tables' shared memory bounds, times the SMs of the current device).  Measured on H100 (profiles/README.md): fewer active
// lanes shorten each warp's divergent serial chain, and a second wave of CTAs costs a whole row's time.
int dd_lanes(int rows)
{
#ifdef AVB_HOSTSIM
    (void)rows;
    return 1;
#else
    int dev = 0, sms = 0, per_sm = 0;
    if (cudaGetDevice(&dev) != cudaSuccess || cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess ||
        cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, dd_entropy_kernel, DD_ENTROPY_THREADS, 0) != cudaSuccess || per_sm < 1) {
        cudaGetLastError();
        sms = 132; per_sm = 13;
    }
    const long slots = (long)sms * per_sm, lanes = (rows + slots - 1) / slots;
    return lanes < 1 ? 1 : lanes > DD_ENTROPY_THREADS ? DD_ENTROPY_THREADS : (int)lanes;
#endif
}

int dd_launch(const DdLaunch &L, int m, cudaStream_t st)
{
    const char *where = "ff_dnxhd_decode_frames_cuda";
    int rows = 0, nblk[2] = { 0, 0 };
    for (int k = 0; k < m; k++) {
        const DdFrame &F = L.f[k];
        rows = rows > F.rows ? rows : F.rows;
        for (int u = 0; u < F.nu; u++) {
            const int b = F.u[u].mbh * F.mbw * (F.is444 ? 12 : 8);
            nblk[u] = nblk[u] > b ? nblk[u] : b;
        }
    }
    if (rows) {
        AVB_LAUNCH(dd_entropy_kernel, dim3((unsigned)((rows + L.lanes - 1) / L.lanes), m), dim3(DD_ENTROPY_THREADS), 0, st)(L);
        if (check_launch(where)) return -1;
    }
    for (int u = 0; u < 2; u++) {
        if (!nblk[u]) continue;
        AVB_LAUNCH(dd_put_kernel, dim3((unsigned)((nblk[u] + 127) / 128), m), dim3(128), 0, st)(L, u);
        if (check_launch(where)) return -1;
    }
    return 0;
}

size_t dd_workspace(const FFDnxhdDecodeWork *works, int n, const FFDnxhdCidEntry *cids, int n_cids)
{
    if (!works || n < 1) return 0;
    size_t total = 0;
    for (int k = 0; k < n; k++) {
        DdFrame F;
        if (dd_frame(works[k], cids, n_cids, F, false)) return 0;
        total += dd_bytes(F);
    }
    return total;
}

}  // namespace
}  // namespace avb

using namespace avb;

extern "C" {

int ff_dnxhd_probe_cuda(const uint8_t *pkt, int size, const FFDnxhdCidEntry *cids, int n_cids, FFDnxhdFrameInfo *info)
{
    if (!info) return dd_refuse("ff_dnxhd_probe_cuda", "NULL info");
    DdUnit u[2];
    int nu = 0;
    return dd_probe(pkt, size, cids, n_cids, *info, u, nu, nullptr, "ff_dnxhd_probe_cuda");
}

size_t ff_dnxhd_decode_workspace_cuda(const FFDnxhdDecodeWork *works, int n, const FFDnxhdCidEntry *cids, int n_cids)
{
    return dd_workspace(works, n, cids, n_cids);
}

int ff_dnxhd_decode_frames_cuda(const FFDnxhdDecodeWork *works, int n, const FFDnxhdCidEntry *cids, int n_cids, void *workspace,
                                size_t workspace_bytes, void *stream)
{
    avb::enter();
    const char *where = "ff_dnxhd_decode_frames_cuda";
    if (n == 0) return 0;
    if (!works || n < 0) return dd_refuse(where, "NULL works or a negative count");
    std::vector<DdFrame> frames(n);
    size_t need = 0;
    for (int k = 0; k < n; k++) {                         // every packet is checked before anything is launched
        if (dd_frame(works[k], cids, n_cids, frames[k], false)) return -1;
        need += dd_bytes(frames[k]);
    }
    if (!workspace || workspace_bytes < need) return dd_refuse(where, "workspace missing or smaller than ff_dnxhd_decode_workspace_cuda returns");
    for (int k = 0; k < n; k++)
        if (dd_frame(works[k], cids, n_cids, frames[k], true)) return -1;
    uint8_t *ws = (uint8_t *)workspace;
    for (int k = 0; k < n; k++) {
        DdFrame &F = frames[k];
        F.coef = reinterpret_cast<int16_t *>(ws);
        ws += dd_align(dd_coef_bytes(F));
        F.ilmb = ws;
        ws += dd_align((size_t)F.rows * F.mbw);
    }
    for (int g0 = 0; g0 < n; g0 += DD_FRAMES_PER_LAUNCH) {
        const int m = n - g0 < DD_FRAMES_PER_LAUNCH ? n - g0 : DD_FRAMES_PER_LAUNCH;
        DdLaunch L;
        memset(&L, 0, sizeof(L));
        int rows = 0;
        for (int k = 0; k < m; k++) { L.f[k] = frames[g0 + k]; rows += L.f[k].rows; }
        L.lanes = dd_lanes(rows);
        if (dd_launch(L, m, (cudaStream_t)stream)) return -1;
    }
    return 0;
}

}  // extern "C"
