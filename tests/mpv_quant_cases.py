"""Shared cases for the mpegvideo encoders' quantiser stage (include/avdsp_b200.h ff_mpv_dct_quantize_batch_cuda): quantiser states, VLC
length tables, blocks fetched from pixel planes, per-block records, and the runners: the reference (oracle/_ref/libmpvqref.so,
ref_mpvq_batch: mpegvideo_enc.c's own static quantisers on a context), its plain-C restatement (oracle/port/orc_mpvq.c), the product compiled
for the host (tests/hostsim/mpv_quant_hostsim.cpp) and the product on the GPU."""
import ctypes as C

import numpy as np

from oracle import loader
from oracle.loader import OrcEncState

REC = np.dtype([("qscale", np.uint8), ("intra", np.uint8), ("dc_scale", np.uint8), ("chroma", np.uint8), ("lambda2", np.uint32)])
FMT_MPEG1, FMT_H261, FMT_H263, FMT_MJPEG = 0, 1, 2, 3
SCORE_UNSET = -123456789            # what coded_score holds before a call: the C code leaves it where it does not write it
BW = 64                             # blocks per row in the pixel planes


# ------------------------------------------------------------------------------------------------------------------------------ tables

class Vlc:
    """VLC length tables shaped like a codec's uni_*_rl_len ([run * 128 + level + 64]); tie = few distinct lengths, which forces equal
    scores between candidates and survivors (the strict-< order decides)"""

    def __init__(self, seed, tie=False):
        rng = np.random.default_rng(seed)
        lo, hi = (4, 6) if tie else (2, 30)
        self.t = [rng.integers(lo, hi, 64 * 128, dtype=np.uint8) for _ in range(4)]
        self.ptrs = (C.c_void_p * 4)(*[t.ctypes.data for t in self.t])

    def product(self):
        from libav_b200 import tables
        v = tables.FFMECmpVlcTables()
        v.intra_ac_vlc_length, v.intra_ac_vlc_last_length, v.inter_ac_vlc_length, v.inter_ac_vlc_last_length = [t.ctypes.data for t in self.t]
        v.luma_dc_vlc_length = None
        return v


def make_state(checker, fdct=0, out_format=FMT_MPEG1, mpeg_quant=0, h263_aic=0, ibias=96, nbias=0, esc=24, maxq=255, elim=(0, 0),
               alt=0, matrices="flat", seed=0):
    """FFMpvQuantState with q matrices for every qscale from the checker's ff_convert_matrix (ref) or its restatement (port)"""
    from libav_b200 import tables
    rng = np.random.default_rng(500 + seed)
    if matrices == "flat":
        im, nm = np.full(64, 16, np.uint16), np.full(64, 16, np.uint16)
    elif matrices == "small":                         # tiny steps: |block * qmat| passes 2^31 at low qscale, levels far past the VLC range
        im, nm = rng.integers(1, 4, 64).astype(np.uint16), rng.integers(1, 4, 64).astype(np.uint16)
    else:
        im, nm = rng.integers(8, 84, 64).astype(np.uint16), rng.integers(8, 64, 64).astype(np.uint16)
    im[0] = 8
    st = tables.FFMpvQuantState()
    st.fdct, st.out_format, st.mpeg_quant, st.h263_aic = fdct, out_format, mpeg_quant, h263_aic
    st.intra_quant_bias, st.inter_quant_bias, st.ac_esc_length = ibias, nbias, esc
    st.min_qcoeff, st.max_qcoeff = -maxq, maxq
    st.luma_elim_threshold, st.chroma_elim_threshold = elim
    o = OrcEncState()
    o.fdct_sel, o.alternate_scan = fdct, alt
    for i in range(64):
        o.intra_matrix[i], o.inter_matrix[i] = int(im[i]), int(nm[i])
        st.intra_matrix[i], st.inter_matrix[i] = int(im[i]), int(nm[i])
    qi, qn, scan = np.zeros(64, np.int32), np.zeros(64, np.int32), np.zeros(64, np.uint8)
    for q in range(1, 32):
        o.qscale = q
        checker.enc_qmatrices(C.byref(o), qi.ctypes.data, qn.ctypes.data, scan.ctypes.data)
        C.memmove(C.addressof(st.q_intra_matrix[q]), qi.ctypes.data, 256)
        C.memmove(C.addressof(st.q_inter_matrix[q]), qn.ctypes.data, 256)
    C.memmove(C.addressof(st.scantable), scan.ctypes.data, 64)
    return st


def states(checker):
    """(label, state): every out_format, mpeg_quant, h263_aic, both transforms, biases of both signs, flat / random / tiny matrices, zigzag
    and alternate scan, the four max_qcoeff ranges the codecs use, elimination thresholds positive, negative and 0"""
    out = []
    k = 0
    for fmt in (FMT_MPEG1, FMT_H263, FMT_MJPEG, FMT_H261):
        for fdct in (0, 2):
            for variant in range(3):
                k += 1
                mq = int(fmt == FMT_H263 and variant == 1)
                aic = int(fmt == FMT_H263 and variant == 2)
                out.append(("fmt%d_fdct%d_v%d" % (fmt, fdct, variant), make_state(
                    checker, fdct, fmt, mq, aic,
                    ibias=(96, 0, -40)[variant], nbias=(0, -64, 50)[variant], esc=(24, 30, 18)[variant],
                    maxq=(127, 255, 1023, 2047)[k % 4], elim=((0, 0), (4, 7), (-3, -5))[(k + variant) % 3],
                    alt=int(variant == 1 and fmt == FMT_MPEG1), matrices=("flat", "random", "small")[(variant + fdct) % 3], seed=k)))
    return out


# ------------------------------------------------------------------------------------------------------------------------------ blocks

KINDS = ("noise", "flat", "sparse", "single", "checker", "escape", "dc_only")


def planes(n, seed, kinds=KINDS):
    """two 8-bit planes holding n 8x8 blocks (BW per row, a 16-byte pad at each row's end) and their offsets; block i's kind is
    kinds[i % len(kinds)].  cur - ref is the inter difference (diff_pixels), cur alone the intra samples (get_pixels)."""
    rng = np.random.default_rng(seed)
    rows = (n + BW - 1) // BW
    stride = BW * 8 + 16
    cur = rng.integers(0, 256, (rows * 8, stride), dtype=np.uint8)
    ref = rng.integers(0, 256, (rows * 8, stride), dtype=np.uint8)
    yy, xx = np.mgrid[0:8, 0:8]
    for i in range(n):
        kind = kinds[i % len(kinds)]
        y, x = (i // BW) * 8, (i % BW) * 8
        r = rng.integers(0, 256, (8, 8))
        if kind == "noise":
            c = r
        elif kind == "flat":
            v = int(rng.integers(0, 256)); c = np.full((8, 8), v); r = np.full((8, 8), v + int(rng.integers(-2, 3)))
        elif kind == "sparse":
            r = np.full((8, 8), 128); c = r.copy()
            for _ in range(int(rng.integers(1, 4))):
                c[rng.integers(0, 8), rng.integers(0, 8)] += int(rng.integers(-60, 61))
        elif kind == "single":                              # one cosine: a single strong coefficient
            u, v = rng.integers(0, 8, 2)
            amp = int(rng.integers(8, 120))
            c = 128 + np.round(amp * np.cos((2 * xx + 1) * u * np.pi / 16) * np.cos((2 * yy + 1) * v * np.pi / 16)).astype(int); r = np.full((8, 8), 128)
        elif kind == "checker":                             # +-255 differences: the largest levels, overflow and clipping
            m = (xx + yy) & 1
            c = np.where(m, 255, 0); r = np.where(m, 0, 255)
            if rng.integers(0, 2):
                c, r = r, c
        elif kind == "escape":                              # strong low frequencies: |level| > 63 at low qscale
            c = np.clip(xx * int(rng.integers(10, 32)) + yy * int(rng.integers(-31, 32)) + int(rng.integers(0, 40)), 0, 255); r = np.zeros((8, 8), int)
        else:                                               # dc_only: a constant difference
            r = rng.integers(40, 200, (8, 8)); c = r + int(rng.integers(-24, 25))
        cur[y:y + 8, x:x + 8] = np.clip(c, 0, 255)
        ref[y:y + 8, x:x + 8] = np.clip(r, 0, 255)
    off = np.array([(i // BW) * 8 * stride + (i % BW) * 8 for i in range(n)], np.uint32)
    return cur, ref, off, stride


def spatial(cur, ref, off, stride, inter=True):
    """the int16 blocks get_pixels (inter False) / diff_pixels (True) leave"""
    n = len(off)
    a, b = cur.reshape(-1), ref.reshape(-1)
    idx = (off[:, None] + (np.arange(8)[:, None] * stride + np.arange(8)[None, :]).reshape(1, 64)).astype(np.int64)
    blk = a[idx].astype(np.int16)
    if inter:
        blk = blk - b[idx].astype(np.int16)
    return np.ascontiguousarray(blk.reshape(n, 64))


def records(n, seed, qscales=range(1, 32), intra=None, lambda2=None):
    """per-block records: qscale cycling through `qscales`, intra / inter mixed (or fixed), dc scales of luma and chroma, lambda2 from 0 to
    large, chroma = block index >= 4 of its macroblock"""
    rng = np.random.default_rng(seed)
    r = np.zeros(n, REC)
    qs = list(qscales)
    r["qscale"] = [qs[i % len(qs)] for i in range(n)]
    r["intra"] = rng.integers(0, 2, n) if intra is None else intra
    r["chroma"] = (np.arange(n) % 6) >= 4
    r["dc_scale"] = np.where(r["chroma"], rng.integers(1, 9, n), rng.choice([1, 2, 4, 8, 13, 24, 46], n))
    if lambda2 is None:
        lam = rng.choice([0, 1, 7, 90, 1000, 20000, 300000, 8000000], n)
        r["lambda2"] = lam.astype(np.uint32)
    else:
        r["lambda2"] = lambda2
    return r


class NR:
    """noise-reduction arrays: dct_offset [2][64], dct_error_sum [2][64], dct_count [2] with non-zero starting sums"""

    def __init__(self, seed):
        rng = np.random.default_rng(seed)
        self.offset = rng.integers(0, 40, 128).astype(np.uint16)
        self.sum = rng.integers(0, 1000, 128).astype(np.int32)
        self.count = rng.integers(0, 50, 2).astype(np.int32)

    def copy(self):
        c = NR.__new__(NR)
        c.offset, c.sum, c.count = self.offset.copy(), self.sum.copy(), self.count.copy()
        return c


# ------------------------------------------------------------------------------------------------------------------------------ oracles

_ARGS = [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_size_t, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
         C.c_void_p, C.c_void_p, C.c_void_p]


class Oracle:
    def __init__(self, fn, name):
        fn.restype = C.c_int
        fn.argtypes = _ARGS
        self.fn, self.name = fn, name

    def run(self, st, vlc, trellis, recs, blocks, nr=None, post=True):
        """blocks: int16 (n, 64) spatial samples.  Returns (levels, last_index, overflow, coded_score) and updates nr in place."""
        n = len(recs)
        b = np.ascontiguousarray(blocks, np.int16).copy()
        last, ovf = np.zeros(n, np.int32), np.zeros(n, np.int32)
        score = np.full(n, SCORE_UNSET, np.int32)
        r = np.ascontiguousarray(recs)
        rc = self.fn(C.byref(st), vlc.ptrs if vlc else None, trellis, int(post), r.ctypes.data, n, b.ctypes.data, last.ctypes.data,
                     ovf.ctypes.data, score.ctypes.data, nr.offset.ctypes.data if nr else None, nr.sum.ctypes.data if nr else None,
                     nr.count.ctypes.data if nr else None)
        assert rc == 0
        return b, last, ovf, score


def ref_oracle():
    """the reference's quantisers, or None where oracle/_ref was not built"""
    lib = loader.ref_lib("mpvq")
    if lib is None:
        return None
    o = Oracle(lib.ref_mpvq_batch, "ref")
    o.lib = lib
    return o


def port_oracle():
    return Oracle(loader.port().lib.orc_mpvq_batch, "port")


def checker():
    """the strongest checker available: the compiled reference where it was built, else the port (which the CPU suite pins to it)"""
    return ref_oracle() or port_oracle()


def matrices_checker():
    """the ff_convert_matrix the q matrices come from: the reference's where it was built, else its restatement"""
    return loader.ref() or loader.port()


# ------------------------------------------------------------------------------------------------------------------------------ product

def nr_struct(offset_ptr, sum_ptr, count_ptr):
    from libav_b200 import tables
    s = tables.FFMpvNoiseReduction()
    s.dct_offset, s.dct_error_sum, s.dct_count = offset_ptr, sum_ptr, count_ptr
    return s


def run_sim(lib, st, vlc, trellis, recs, blocks=None, pix=None, nr=None):
    """the host-compiled product: blocks (n, 64) spatial samples (the slot path), or pix = (cur, ref or None, off, stride) (the fused
    front end).  Returns (levels, last_index, coded_score) and updates nr in place."""
    n = len(recs)
    h = lib.ff_mpv_quant_state_cuda(C.byref(st), C.byref(vlc.product()) if vlc else None)
    assert h, lib.avb200_last_error()
    try:
        out = np.zeros((n, 64), np.int16) if blocks is None else np.ascontiguousarray(blocks, np.int16).copy()
        last = np.full(n, -7, np.int32)
        score = np.full(n, SCORE_UNSET, np.int32)
        r = np.ascontiguousarray(recs)
        nrs = nr_struct(nr.offset.ctypes.data, nr.sum.ctypes.data, nr.count.ctypes.data) if nr else None
        if pix is None:
            args = (None, None, None, None, 0)
        else:
            cur, ref, off, stride = pix
            args = (cur.ctypes.data, ref.ctypes.data if ref is not None else None, off.ctypes.data, None, stride)
        rc = lib.ff_mpv_dct_quantize_batch_cuda(h, trellis, r.ctypes.data, *args, out.ctypes.data, n, last.ctypes.data, score.ctypes.data,
                                                C.byref(nrs) if nr else None, None)
        assert rc == 0, lib.avb200_last_error()
        return out, last, score
    finally:
        lib.ff_mpv_quant_state_free_cuda(h)


def undefined_blocks(st, vlc, trellis, recs, blocks, nr=None):
    """the blocks whose trellis result depends on table entries the reference never writes (scores that wrap past 2^31 so that no candidate
    beats the initial best score): the port run with two different table fillings disagrees on exactly those"""
    if not trellis:
        return np.zeros(len(recs), bool)
    fill = loader.port().lib.orc_mpvq_set_table_fill
    port = port_oracle()
    out = []
    for v in (0, 0x5a5a5a5):
        fill(v)
        out.append(port.run(st, vlc, trellis, recs, blocks, nr.copy() if nr else None))
    fill(0)
    a, b = out
    return (a[0] != b[0]).any(axis=1) | (a[1] != b[1]) | (a[3] != b[3])


def compare(label, want, got_levels, got_last, got_score, trellis, skip=None):
    """skip: blocks left out (undefined_blocks)"""
    levels, last, _, score = want
    diff = (levels != got_levels).any(axis=1) | (last != got_last) | ((score != got_score) if trellis else False)
    if skip is not None:
        diff &= ~skip
    bad = np.nonzero(diff)[0]
    assert len(bad) == 0, (label, len(bad), int(bad[0]), levels[bad[0]].tolist(), got_levels[bad[0]].tolist(), int(last[bad[0]]),
                           int(got_last[bad[0]]), int(score[bad[0]]), int(got_score[bad[0]]))


def alternate_scan_recompute(levels, last, scantable):
    """encode_mb_internal's recompute of block_last_index for a non-C quantiser under alternate_scan (mpegvideo_enc.c:2312-2325)"""
    out = last.copy()
    for i in range(len(last)):
        if last[i] > 0:
            j = 63
            while j > 0 and not levels[i][scantable[j]]:
                j -= 1
            out[i] = j
    return out
