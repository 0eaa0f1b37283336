// libav_b200/csrc/prores_dec.cu -- the ProRes decoder (libavcodec/proresdec.c: decode_frame) as one batched call: n packets to n frames,
// every sample the reference decoder writes written with its value.
//
// Every slice plane (at most 8 macroblocks) is an independent serial chain: decode_slice_plane starts a fresh reader at the plane's first
// byte, and decode_slice's scale factor and the frame's matrices are all a slice needs.  Stages, per launch of up to 64 packets:
//   offsets  one thread per (packet, picture, 32 slices): the sum of the chunk's be16 slice sizes, then one thread per chunk again: the
//            slices' offsets from the picture's first slice, from the chunk sums before it.  The host checks the table but uploads nothing.
//   entropy  one thread per (packet, picture, plane, slice), Y planes first: the slice header, the plane's blocks zeroed, then its DC and
//            AC coefficients into the workspace in the order ff_prores_decode_pictures_cuda takes, and the plane's status; the Y thread
//            also records the slice's FFProresSlice.  A warp has `lanes` active threads: at most 8, fewer when that keeps every CTA
//            resident (prd_lanes).
//   alpha    one thread per (packet, picture, slice) of a format with alpha: unpack_alpha straight into the alpha plane when Y, U and V
//            decoded and the slice has alpha bytes.  One-warp CTAs with `alpha_lanes` active threads: all 32 (prd_alpha_lanes).
//   put      prores.cu's picture kernels (launch_prores_pictures), which skip the planes a slice does not write.
// The kernels' threads never communicate, so the file also compiles as host C++ for tests/hostsim/.
#include "common.cuh"
#include "prores_dec.cuh"
#include "../../include/avdsp_b200.h"
#include <string.h>
#include <vector>

namespace avb {
namespace {

constexpr int PRD_FRAMES_PER_LAUNCH = 64;       // one launch per stage for a call of up to 64 packets
#ifdef AVB_HOSTSIM
constexpr int PRD_THREADS = 1;
#else
constexpr int PRD_THREADS = 32;
#endif
constexpr int PRD_INVALIDDATA = -0x3ebbb1b7;     // AVERROR_INVALIDDATA
constexpr uint32_t PRD_FRAME_ID = 0x69637066u;  // 'icpf'
struct PrdLaunch { PrdFrame f[PRD_FRAMES_PER_LAUNCH]; int lanes, alpha_lanes; };
static_assert(sizeof(PrdLaunch) <= 32764, "kernel parameters");

__device__ __forceinline__ uint32_t prd_be16(const PrdFrame &F, uint32_t o) { return F.pkt[o] << 8 | F.pkt[o + 1]; }

// ---- kernels ------------------------------------------------------------------------------------------------------------------------------
// thread -> (picture, chunk) of a packet; false past its chunks
__device__ __forceinline__ bool prd_chunk_of(const PrdFrame &F, int t, int &p, int &c)
{
    for (p = 0; p < F.npics; p++) {
        const int nc = (F.pic[p].n_slices + PRD_CHUNK - 1) / PRD_CHUNK;
        if (t < nc) { c = t; return true; }
        t -= nc;
    }
    return false;
}

__global__ void __launch_bounds__(128) prd_chunk_kernel(const __grid_constant__ PrdLaunch L)
{
    const PrdFrame &F = L.f[blockIdx.y];
    int p, c;
    if (!prd_chunk_of(F, (int)(blockIdx.x * blockDim.x + threadIdx.x), p, c)) return;
    const PrdPic &P = F.pic[p];
    const int s1 = min(P.n_slices, (c + 1) * PRD_CHUNK);
    uint32_t sum = 0;
    for (int s = c * PRD_CHUNK; s < s1; s++) sum += prd_be16(F, P.index + 2 * s);
    P.chunks[c] = sum;
}

__global__ void __launch_bounds__(128) prd_offset_kernel(const __grid_constant__ PrdLaunch L)
{
    const PrdFrame &F = L.f[blockIdx.y];
    int p, c;
    if (!prd_chunk_of(F, (int)(blockIdx.x * blockDim.x + threadIdx.x), p, c)) return;
    const PrdPic &P = F.pic[p];
    uint32_t off = 0;
    for (int k = 0; k < c; k++) off += P.chunks[k];
    const int s1 = min(P.n_slices, (c + 1) * PRD_CHUNK);
    for (int s = c * PRD_CHUNK; s < s1; s++) { P.offs[s] = off; off += prd_be16(F, P.index + 2 * s); }
    if (s1 == P.n_slices) P.offs[s1] = off;
}

// one plane of one slice (decode_slice up to its plane, then decode_slice_plane's entropy half)
__device__ inline void prd_plane(const PrdFrame &F, const PrdPic &P, int plane, int s)
{
    const int nxs = pr_slices_per_row(F.mbw, P.swf);
    int row, x, w;
    prd_slice_pos(F.mbw, P.swf, nxs, s, row, x, w);
    const int bpm = prd_bpm(F.c444), ncb = F.c444 ? 4 : 2;
    const uint32_t first = (uint32_t)((row * F.mbw + x) * bpm);
    const uint32_t data = P.index + 2u * (uint32_t)P.n_slices, off = data + P.offs[s];
    const int size = (int)(P.offs[s + 1] - P.offs[s]);
    uint8_t *st = reinterpret_cast<uint8_t *>(P.status + s) + plane;
    int coff[4], sz[4], sf = 1;
    const bool ok = prd_slice_header(F, off, size, coff, sz, sf);
    if (plane == 0) { FFProresSlice sl; sl.first_block = first; sl.sf = (uint16_t)sf; sl.reserved = 0; P.slices[s] = sl; }
    if (!ok) { *st = 0; return; }
    const int nb = plane ? w * ncb : 4 * w;
    int16_t *blk = P.coef + 64 * ((size_t)first + (plane ? 4 * w + (plane - 1) * w * ncb : 0));
    uint4 *b4 = reinterpret_cast<uint4 *>(blk);
    for (int k = 0; k < nb * 8; k++) b4[k] = make_uint4(0, 0, 0, 0);
    PrdBits r;
    prd_bits_init(r, F, off + (uint32_t)coff[plane], sz[plane]);
    prd_dc(r, blk, nb);
    const int swf = 31 - prd_clz((uint32_t)w);                        // av_log2(mbs_per_slice)
    const int psf = plane ? swf + (F.c444 ? 2 : 1) : swf + 2;
    *st = prd_ac(r, blk, nb, psf, pe_scan[F.scan]) < 0 ? 0 : 1;
}

// A CTA is one warp (one thread in the host build) and takes `lanes` consecutive tasks of one packet, one per lane.
__global__ void __launch_bounds__(PRD_THREADS) prd_entropy_kernel(const __grid_constant__ PrdLaunch L)
{
    const PrdFrame &F = L.f[blockIdx.y];
    if ((int)threadIdx.x >= L.lanes) return;
    int t = (int)blockIdx.x * L.lanes + (int)threadIdx.x;
    for (int p = 0; p < F.npics; p++) {
        const int n = F.pic[p].n_slices;
        if (t < 3 * n) { prd_plane(F, F.pic[p], t / n, t % n); return; }
        t -= 3 * n;
    }
}

// A CTA is one warp (one thread in the host build) and takes `alpha_lanes` consecutive slices of one packet, one per lane.
__global__ void __launch_bounds__(PRD_THREADS) prd_alpha_kernel(const __grid_constant__ PrdLaunch L)
{
    const PrdFrame &F = L.f[blockIdx.y];
    if (!F.alpha || (int)threadIdx.x >= L.alpha_lanes) return;
    int s = (int)blockIdx.x * L.alpha_lanes + (int)threadIdx.x, p = 0;
    for (; p < F.npics && s >= F.pic[p].n_slices; p++) s -= F.pic[p].n_slices;
    if (p >= F.npics) return;
    const PrdPic &P = F.pic[p];
    if (!pr_plane_written(P.status[s], 2)) return;
    const uint32_t off = P.index + 2u * (uint32_t)P.n_slices + P.offs[s];
    int coff[4], sz[4], sf;
    if (!prd_slice_header(F, off, (int)(P.offs[s + 1] - P.offs[s]), coff, sz, sf) || !sz[3]) return;
    int row, x, w;
    prd_slice_pos(F.mbw, P.swf, pr_slices_per_row(F.mbw, P.swf), s, row, x, w);
    const ptrdiff_t ls = (ptrdiff_t)F.als << F.il;
    uint8_t *dst = F.adata + (P.field ? F.als : 0) + (ptrdiff_t)(row << 4) * ls + (x << 5);
    PrdBits r;
    prd_bits_init(r, F, off + (uint32_t)coff[3], sz[3]);
    if (F.alpha == 2) prd_alpha<16>(r, dst, ls, w);
    else prd_alpha<8>(r, dst, ls, w);
}

// ---- host side ------------------------------------------------------------------------------------------------------------------------------
int prd_refuse(const char *where, const char *msg) { set_error_msg(where, msg); return -1; }
inline uint32_t prd_rb32(const uint8_t *p) { return (uint32_t)p[0] << 24 | (uint32_t)p[1] << 16 | (uint32_t)p[2] << 8 | p[3]; }
inline int prd_rb16(const uint8_t *p) { return p[0] << 8 | p[1]; }

// what decode_frame derives before and after get_buffer
struct PrdProbe {
    FFProresFrameInfo info;
    int c444, alpha_info, frame_type;
    uint8_t qm[2][64];
    int npics;
    struct { uint32_t index; int n_slices, swf; } pic[2];
    uint8_t *pic_data[3];                        // the caller's Y, U, V planes and frame linesizes
    int pic_ls[3];
};

// decode_picture_header at packet offset `at` with data_size bytes: its return value (pic_data_size, or < 0)
int prd_picture_header(const uint8_t *pkt, uint32_t at, int data_size, int width, int height, int il, PrdProbe &R, int k)
{
    const uint8_t *buf = pkt + at;
    const int hdr = data_size > 0 ? buf[0] >> 3 : 0;
    if (hdr < 8 || hdr > data_size) return PRD_INVALIDDATA;
    const int pic_data_size = (int)prd_rb32(buf + 1);
    if (pic_data_size > data_size) return PRD_INVALIDDATA;
    const int swf = buf[7] >> 4, shf = buf[7] & 15;
    if (swf > 3 || shf) return PRD_INVALIDDATA;
    const int mbw = (width + 15) >> 4, mbh = (height + (1 << (4 + il)) - 1) >> (4 + il);
    const long n = (long)pr_slices_per_row(mbw, swf) * mbh;
    if (n != prd_rb16(buf + 5)) return PRD_INVALIDDATA;
    if (hdr + n * 2 > data_size) return PRD_INVALIDDATA;
    long end = hdr + n * 2;
    for (long s = 0; s < n; s++) end += prd_rb16(buf + hdr + 2 * s);
    if (end > data_size) return PRD_INVALIDDATA;                     // "out of slice data" (-1, which decode_frame turns into this)
    R.pic[k].index = at + (uint32_t)hdr;
    R.pic[k].n_slices = (int)n;
    R.pic[k].swf = swf;
    return pic_data_size;
}

int prd_probe(const uint8_t *pkt, int size, int width, int height, PrdProbe &R, const char *where)
{
    memset(&R, 0, sizeof(R));
    FFProresFrameInfo &info = R.info;
    if (!pkt || size < 0) return prd_refuse(where, "NULL packet or a negative size");
    if (size < 28 || (uint32_t)size < prd_rb32(pkt) || prd_rb32(pkt + 4) != PRD_FRAME_ID) return PRD_INVALIDDATA;
    const uint8_t *buf = pkt + 8;
    int buf_size = size - 8;
    // decode_frame_header (bytes 8..19 are read whatever hdr_size says; size >= 28 keeps them inside the packet)
    const int hdr = prd_rb16(buf);
    if (hdr > buf_size) return PRD_INVALIDDATA;
    if (prd_rb16(buf + 2) >= 2) return PRD_INVALIDDATA;
    if (prd_rb16(buf + 8) != width || prd_rb16(buf + 10) != height) return PRD_INVALIDDATA;
    R.frame_type = (buf[12] >> 2) & 3;
    if (R.frame_type > 2) return PRD_INVALIDDATA;
    const int cf = (buf[12] >> 6) & 3;
    R.alpha_info = buf[17] & 15;
    if (R.alpha_info > 2) return PRD_INVALIDDATA;
    if (cf != 2 && cf != 3) return PRD_INVALIDDATA;
    R.c444 = cf == 3;
    int ptr = 20;
    const int flags = buf[19];
    if (flags & 2) {
        if (ptr > hdr - 64) return PRD_INVALIDDATA;
        memcpy(R.qm[0], buf + ptr, 64);
        ptr += 64;
    } else memset(R.qm[0], 4, 64);
    if (flags & 1) {
        if (ptr > hdr - 64) return PRD_INVALIDDATA;
        memcpy(R.qm[1], buf + ptr, 64);
    } else memset(R.qm[1], 4, 64);
    if (width < 1 || height < 1) return prd_refuse(where, "a zero width or height (get_buffer refuses the frame)");
    const int il = R.frame_type != 0;
    info.pix_fmt = R.c444 ? (R.alpha_info ? FF_PRORES_PIX_FMT_YUVA444P10 : FF_PRORES_PIX_FMT_YUV444P10)
                          : (R.alpha_info ? FF_PRORES_PIX_FMT_YUVA422P10 : FF_PRORES_PIX_FMT_YUV422P10);
    info.interlaced_frame = il;
    info.top_field_first = il ? R.frame_type & 1 : 0;
    info.color_primaries = buf[14]; info.color_trc = buf[15]; info.colorspace = buf[16];
    info.lines = ((height + (1 << (4 + il)) - 1) >> (4 + il)) * 16 << il;
    // get_buffer, then each picture: a header that fails ends the frame with AVERROR_INVALIDDATA after the pictures before it
    uint32_t at = 8 + (uint32_t)hdr;
    buf_size -= hdr;
    info.result = size;
    for (int k = 0; k <= il; k++) {
        const int pds = prd_picture_header(pkt, at, buf_size, width, height, il, R, k);
        if (pds < 0) { info.result = PRD_INVALIDDATA; break; }
        R.npics = k + 1;
        at += (uint32_t)pds;
        buf_size -= pds;
    }
    info.pictures = R.npics;
    return 0;
}

// the checks of one packet and its planes; fills F's geometry (not its workspace pointers) and the picture works' constant part
int prd_frame(const FFProresDecodeWork &w, PrdFrame &F, PrdProbe &R)
{
    const char *where = "ff_prores_decode_frames_cuda";
    memset(&F, 0, sizeof(F));
    const int ret = prd_probe(w.pkt_host, w.size, w.width, w.height, R, where);
    if (ret > 0 || ret < -1) return prd_refuse(where, "a packet the decoder refuses (ff_prores_probe_cuda returns its AVERROR)");
    if (ret) return -1;
    if (!w.pkt) return prd_refuse(where, "NULL device packet");
    const int alpha = R.alpha_info != 0, mbw = (w.width + 15) >> 4;
    for (int p = 0; p < 3 + alpha; p++) {
        if (!w.data[p] || ((uintptr_t)w.data[p] & 1)) return prd_refuse(where, p == 3 ? "NULL or odd alpha plane" : "NULL or odd plane pointer");
        if (w.linesize[p] <= 0 || (w.linesize[p] & 1) || w.linesize[p] < (long)mbw * (p == 1 || p == 2 ? (R.c444 ? 32 : 16) : 32))
            return prd_refuse(where, "linesize must be even, positive and at least the width of whole macroblocks");
        if (w.lines[p] < R.info.lines) return prd_refuse(where, "a plane holds fewer lines than the frame needs");
    }
    F.pkt = w.pkt; F.size = (uint32_t)w.size;
    F.mbw = mbw; F.mbh = R.info.lines >> (4 + R.info.interlaced_frame);
    F.c444 = R.c444; F.alpha = R.alpha_info;
    F.il = R.info.interlaced_frame; F.scan = F.il;
    F.npics = R.npics;
    F.adata = alpha ? w.data[3] : nullptr; F.als = alpha ? w.linesize[3] : 0;
    for (int k = 0; k < R.npics; k++) {
        F.pic[k].index = R.pic[k].index; F.pic[k].n_slices = R.pic[k].n_slices; F.pic[k].swf = R.pic[k].swf;
        F.pic[k].field = F.il && k == R.info.top_field_first;           // !(pic_num ^ top_field_first)
    }
    return 0;
}

size_t prd_align(size_t v) { return (v + 255) & ~(size_t)255; }
size_t prd_pic_bytes(const PrdFrame &F, const PrdPic &P)
{
    const size_t n = (size_t)P.n_slices, chunks = (n + PRD_CHUNK - 1) / PRD_CHUNK;
    return prd_align((size_t)F.mbw * F.mbh * prd_bpm(F.c444) * 128) + prd_align(n * sizeof(FFProresSlice)) + prd_align(n * 4) +
           prd_align((n + 1) * 4) + prd_align(chunks * 4);
}
size_t prd_bytes(const PrdFrame &F)
{
    size_t b = 0;
    for (int k = 0; k < F.npics; k++) b += prd_pic_bytes(F, F.pic[k]);
    return b;
}
void prd_place(PrdFrame &F, uint8_t *&ws)
{
    for (int k = 0; k < F.npics; k++) {
        PrdPic &P = F.pic[k];
        const size_t n = (size_t)P.n_slices;
        P.coef = reinterpret_cast<int16_t *>(ws); ws += prd_align((size_t)F.mbw * F.mbh * prd_bpm(F.c444) * 128);
        P.slices = reinterpret_cast<FFProresSlice *>(ws); ws += prd_align(n * sizeof(FFProresSlice));
        P.status = reinterpret_cast<uint32_t *>(ws); ws += prd_align(n * 4);
        P.offs = reinterpret_cast<uint32_t *>(ws); ws += prd_align((n + 1) * 4);
        P.chunks = reinterpret_cast<uint32_t *>(ws); ws += prd_align((n + PRD_CHUNK - 1) / PRD_CHUNK * 4);
    }
}

// Active lanes per entropy warp for a launch of `tasks` slice planes: the fewest that still fit every CTA on the device at once (resident
// one-warp CTAs per SM times the SMs of the current device), and never more than PRD_MAX_LANES.  Measured on H100 (profiles/README.md):
// the planes' serial chains differ in length, so a warp runs as long as its longest lane, and 8 lanes in more waves beat 32 lanes in one
// (6.2 against 8.3 ms for 64 1080p HQ packets).  The test knob prd_lanes overrides it for the launch-shape sweep.
constexpr int PRD_MAX_LANES = 8;
int prd_lanes(long tasks)
{
#ifdef AVB_HOSTSIM
    (void)tasks;
    return 1;
#else
    const int forced = tuning("prd_lanes");
    if (forced >= 1 && forced <= PRD_THREADS) return forced;
    int per_sm = 0;
    if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, prd_entropy_kernel, PRD_THREADS, 0) != cudaSuccess || per_sm < 1) {
        cudaGetLastError();
        per_sm = 32;
    }
    const long slots = (long)sm_count() * per_sm, lanes = (tasks + slots - 1) / slots;
    return lanes < 1 ? 1 : lanes > PRD_MAX_LANES ? PRD_MAX_LANES : (int)lanes;
#endif
}

// Active lanes per alpha warp: all of them.  Measured on H100 (profiles/README.md): a slice's alpha is one long chain of short codes
// and 2-byte stores, and full warps are the fastest or within 10 % of it (64 1080p 4444 packets: 6.6 ms per call at 32 lanes, 10.5 at 8).
// The test knob prd_alpha_lanes overrides it for the launch-shape sweep.
int prd_alpha_lanes()
{
#ifdef AVB_HOSTSIM
    return 1;
#else
    const int forced = tuning("prd_alpha_lanes");
    return forced >= 1 && forced <= PRD_THREADS ? forced : PRD_THREADS;
#endif
}

int prd_launch(PrdLaunch &L, int m, const PrdProbe *probes, cudaStream_t st)
{
    const char *where = "ff_prores_decode_frames_cuda";
    long chunks = 0, tasks = 0, slices = 0, all_tasks = 0;
    for (int k = 0; k < m; k++) {
        long c = 0, s = 0;
        for (int p = 0; p < L.f[k].npics; p++) { c += (L.f[k].pic[p].n_slices + PRD_CHUNK - 1) / PRD_CHUNK; s += L.f[k].pic[p].n_slices; }
        chunks = chunks > c ? chunks : c;
        slices = slices > s ? slices : s;
        tasks = tasks > 3 * s ? tasks : 3 * s;
        all_tasks += 3 * s;
    }
    if (!tasks) return 0;
    L.lanes = prd_lanes(all_tasks);
    AVB_LAUNCH(prd_chunk_kernel, dim3((unsigned)((chunks + 127) / 128), m), dim3(128), 0, st)(L);
    if (check_launch(where)) return -1;
    AVB_LAUNCH(prd_offset_kernel, dim3((unsigned)((chunks + 127) / 128), m), dim3(128), 0, st)(L);
    if (check_launch(where)) return -1;
    AVB_LAUNCH(prd_entropy_kernel, dim3((unsigned)((tasks + L.lanes - 1) / L.lanes), m), dim3(PRD_THREADS), 0, st)(L);
    if (check_launch(where)) return -1;
    long alpha_slices = 0;
    for (int k = 0; k < m; k++)
        for (int p = 0; p < L.f[k].npics && L.f[k].alpha; p++) alpha_slices += L.f[k].pic[p].n_slices;
    if (alpha_slices) {
        L.alpha_lanes = prd_alpha_lanes();
        AVB_LAUNCH(prd_alpha_kernel, dim3((unsigned)((slices + L.alpha_lanes - 1) / L.alpha_lanes), m), dim3(PRD_THREADS), 0, st)(L);
        if (check_launch(where)) return -1;
    }
    std::vector<FFProresPictureWork> pics;
    std::vector<const uint32_t *> status;
    for (int k = 0; k < m; k++) {
        const PrdFrame &F = L.f[k];
        for (int p = 0; p < F.npics; p++) {
            FFProresPictureWork w;
            memset(&w, 0, sizeof(w));
            for (int c = 0; c < 3; c++) {
                w.data[c] = probes[k].pic_data[c] + (F.pic[p].field ? probes[k].pic_ls[c] : 0);
                w.linesize[c] = probes[k].pic_ls[c] << F.il;
                w.mb_rows[c] = F.mbh;
            }
            w.mb_width = F.mbw; w.mb_height = F.mbh;
            w.slice_width_factor = F.pic[p].swf;
            w.chroma_format = F.c444 ? 3 : 2;
            memcpy(w.qmat_luma, probes[k].qm[0], 64); memcpy(w.qmat_chroma, probes[k].qm[1], 64);
            w.slices = F.pic[p].slices; w.n_slices = F.pic[p].n_slices;
            w.blocks = F.pic[p].coef; w.n_blocks = (size_t)F.mbw * F.mbh * prd_bpm(F.c444);
            pics.push_back(w);
            status.push_back(F.pic[p].status);
        }
    }
    return launch_prores_pictures(pics.data(), (int)pics.size(), st, status.data());
}

}  // namespace
}  // namespace avb

using namespace avb;

extern "C" {

int ff_prores_probe_cuda(const uint8_t *pkt, int size, int width, int height, FFProresFrameInfo *info)
{
    if (!info) return prd_refuse("ff_prores_probe_cuda", "NULL info");
    PrdProbe R;
    const int ret = prd_probe(pkt, size, width, height, R, "ff_prores_probe_cuda");
    *info = R.info;
    return ret;
}

size_t ff_prores_decode_workspace_cuda(const FFProresDecodeWork *works, int n)
{
    if (!works || n < 1) return 0;
    size_t total = 0;
    for (int k = 0; k < n; k++) {
        PrdFrame F;
        PrdProbe R;
        if (prd_frame(works[k], F, R)) return 0;
        total += prd_bytes(F);
    }
    return total;
}

int ff_prores_decode_frames_cuda(const FFProresDecodeWork *works, int n, void *workspace, size_t workspace_bytes, void *stream)
{
    avb::enter();
    const char *where = "ff_prores_decode_frames_cuda";
    if (n == 0) return 0;
    if (!works || n < 0) return prd_refuse(where, "NULL works or a negative count");
    std::vector<PrdFrame> frames(n);
    std::vector<PrdProbe> probes(n);
    size_t need = 0;
    for (int k = 0; k < n; k++) {                         // every packet is checked before anything is launched
        if (prd_frame(works[k], frames[k], probes[k])) return -1;
        need += prd_bytes(frames[k]);
    }
    if (!workspace || workspace_bytes < need) return prd_refuse(where, "workspace missing or smaller than ff_prores_decode_workspace_cuda returns");
    if ((uintptr_t)workspace & 15) return prd_refuse(where, "workspace not 16-byte aligned (the coefficient blocks are zeroed 16 bytes at a time)");
    uint8_t *ws = (uint8_t *)workspace;
    for (int k = 0; k < n; k++) {
        prd_place(frames[k], ws);
        for (int c = 0; c < 3; c++) { probes[k].pic_data[c] = works[k].data[c]; probes[k].pic_ls[c] = works[k].linesize[c]; }
    }
    for (int g0 = 0; g0 < n; g0 += PRD_FRAMES_PER_LAUNCH) {
        const int m = n - g0 < PRD_FRAMES_PER_LAUNCH ? n - g0 : PRD_FRAMES_PER_LAUNCH;
        PrdLaunch L;
        memset(&L, 0, sizeof(L));
        for (int k = 0; k < m; k++) L.f[k] = frames[g0 + k];
        if (prd_launch(L, m, probes.data() + g0, (cudaStream_t)stream)) return -1;
    }
    return 0;
}

}  // extern "C"
