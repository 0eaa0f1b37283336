"""CPU: the mpegvideo encoders' quantiser stage (libav_b200/csrc/mpv_quant.cu + mpv_quant.cuh) compiled for the host
(tests/hostsim/mpv_quant_hostsim.cpp) against the reference's own quantisers (libavcodec/mpegvideo_enc.c: ff_dct_quantize_c,
dct_quantize_trellis_c, denoise_dct_c, clip_coeffs, dct_single_coeff_elimination; oracle/_ref/libmpvqref.so), and the plain-C port
(oracle/port/orc_mpvq.c) against the same reference.  Every output is compared: levels, block_last_index, overflow, coded_score and the
noise-reduction sums and counts.  States cover every out_format, mpeg_quant, h263_aic, islow / ifast, biases of both signs, flat / random /
tiny matrices, zigzag and alternate scan, max_qcoeff 127 / 255 / 1023 / 2047, elimination thresholds positive / negative / 0; blocks are noise,
flat, sparse, single-coefficient, +-255 checkerboards, escape-range and DC-only differences at every qscale, intra and inter, luma and
chroma, lambda2 from 0 to 8e6, with random and tie-forcing VLC tables, noise reduction on and off.  Also: the dct_quantize slots on a live
context, the hook's refusals and its place in the reference glue, the batch call's refusals, and the struct layouts."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

import mpv_quant_cases as M

ROOT = M.ROOT


@pytest.fixture(scope="session")
def mats(built):
    return M.matrices_checker()


@pytest.fixture(scope="session")
def ref(built):
    r = M.ref_oracle()
    if r is None:
        pytest.skip("the reference was not built (oracle/_ref)")
    return r


@pytest.fixture(scope="session")
def sim(built):
    return M.sim_lib()


def _cases(mats, n=420, seed=0):
    """(label, state, vlc, trellis, recs, blocks, nr) over every state, both quantisers, noise reduction on and off"""
    out = []
    for k, (label, st) in enumerate(M.states(mats)):
        for trellis in (0, 1):
            cur, rf, off, stride = M.planes(n, seed + 31 * k + trellis)
            inter = bool(k % 2)
            blk = M.spatial(cur, rf, off, stride, inter=inter)
            recs = M.records(n, seed + 7 * k + trellis)
            vlc = M.Vlc(k, tie=bool(k % 3 == 1))
            out.append(("%s_trellis%d" % (label, trellis), st, vlc, trellis, recs, blk, M.NR(k) if k % 2 == 0 else None))
    return out


def test_port_equals_reference(mats, ref):
    port = M.port_oracle()
    for label, st, vlc, trellis, recs, blk, nr in _cases(mats):
        for post in (True, False):
            nr1, nr2 = (nr.copy(), nr.copy()) if nr else (None, None)
            want = ref.run(st, vlc, trellis, recs, blk, nr1, post)
            got = port.run(st, vlc, trellis, recs, blk, nr2, post)
            skip = M.undefined_blocks(st, vlc, trellis, recs, blk, nr)
            assert skip.sum() < len(recs) // 20, (label, int(skip.sum()))
            for name, a, b in zip(("levels", "last_index", "overflow", "coded_score"), want, got):
                d = (a != b).reshape(len(recs), -1).any(axis=1) & ~skip
                assert not d.any(), (label, post, name, np.nonzero(d)[0][:5])
            if nr:
                assert np.array_equal(nr1.sum, nr2.sum) and np.array_equal(nr1.count, nr2.count), label


def test_hostsim_equals_reference(mats, sim):
    """the kernel body (host C++) through ff_mpv_dct_quantize_batch_cuda, the slot path (blocks hold the spatial samples), against the
    strongest checker; the checker's overflow flags must have led to clipping somewhere"""
    chk = M.checker()
    clipped = escapes = 0
    for label, st, vlc, trellis, recs, blk, nr in _cases(mats):
        nr1, nr2 = (nr.copy(), nr.copy()) if nr else (None, None)
        want = chk.run(st, vlc, trellis, recs, blk, nr1)
        got = M.run_sim(sim, st, vlc, trellis, recs, blocks=blk, nr=nr2)
        M.compare(label, want, *got, trellis, skip=M.undefined_blocks(st, vlc, trellis, recs, blk, nr))
        if nr:
            assert np.array_equal(nr1.sum, nr2.sum) and np.array_equal(nr1.count, nr2.count), label
        clipped += int(want[2].sum())
        escapes += int((np.abs(want[0]) > 63).any(axis=1).sum())
    assert clipped > 100 and escapes > 100


def test_hostsim_fused_equals_unfused(mats, sim):
    """the fused front end (get_pixels / diff_pixels + fdct in the kernel) gives bitwise the result of the same blocks staged first"""
    for label, st in M.states(mats)[::3]:
        cur, rf, off, stride = M.planes(300, 5)
        recs = M.records(300, 6)
        vlc = M.Vlc(2)
        for trellis in (0, 1):
            for inter in (False, True):
                blk = M.spatial(cur, rf, off, stride, inter=inter)
                a = M.run_sim(sim, st, vlc, trellis, recs, blocks=blk)
                b = M.run_sim(sim, st, vlc, trellis, recs, pix=(cur, rf if inter else None, off, stride))
                for x, y in zip(a, b):
                    assert np.array_equal(x, y), (label, trellis, inter)


def test_every_qscale_intra_inter_luma_chroma(mats, sim):
    """one state per transform, every qscale 1..31 in one batch with intra / inter and luma / chroma dc scales, both quantisers"""
    chk = M.checker()
    for fdct in (0, 2):
        st = M.make_state(mats, fdct, M.FMT_MPEG1, matrices="random", seed=40 + fdct, elim=(-2, 3))
        cur, rf, off, stride = M.planes(31 * 12, 9)
        blk = M.spatial(cur, rf, off, stride)
        recs = M.records(31 * 12, 3)
        recs["intra"] = (np.arange(31 * 12) // 31) % 2
        assert set(recs["qscale"]) == set(range(1, 32))
        for trellis in (0, 1):
            M.compare(fdct, chk.run(st, M.Vlc(1), trellis, recs, blk), *M.run_sim(sim, st, M.Vlc(1), trellis, recs, blocks=blk), trellis,
                      skip=M.undefined_blocks(st, M.Vlc(1), trellis, recs, blk))


def test_integer_wrap_cases(mats, sim):
    """levels that make (unquant - dct)^2 and block * qmat pass 2^31 (tiny matrices, qscale 1, +-255 checkerboards and ramps) must wrap
    exactly like the reference"""
    chk = M.checker()
    for fmt in (M.FMT_MPEG1, M.FMT_H263):
        for fdct in (0, 2):
            st = M.make_state(mats, fdct, fmt, matrices="small", maxq=2047, seed=60 + fmt + fdct)
            cur, rf, off, stride = M.planes(400, 11, kinds=("checker", "escape"))
            blk = M.spatial(cur, rf, off, stride)
            recs = M.records(400, 12, qscales=(1, 2), lambda2=np.uint32(1 << 22))
            for trellis in (0, 1):
                want = chk.run(st, M.Vlc(4), trellis, recs, blk)
                assert (np.abs(want[0]) > 1000).any()
                M.compare((fmt, fdct), want, *M.run_sim(sim, st, M.Vlc(4), trellis, recs, blocks=blk), trellis,
                          skip=M.undefined_blocks(st, M.Vlc(4), trellis, recs, blk))


def test_undefined_blocks_are_deterministic(mats, sim):
    """where the reference reads trellis table entries it never wrote (scores wrapped past 2^31), the kernel clears them per position: its
    result on those blocks is the port's with zeroed tables, on both front ends"""
    from oracle import loader
    port = M.port_oracle()
    loader.port().lib.orc_mpvq_set_table_fill(0)
    found = 0
    for label, st, vlc, trellis, recs, blk, nr in _cases(mats):
        if not trellis:
            continue
        undefined = M.undefined_blocks(st, vlc, trellis, recs, blk)
        if not undefined.any():
            continue
        found += int(undefined.sum())
        want = port.run(st, vlc, 1, recs, blk)
        M.compare(label, want, *M.run_sim(sim, st, vlc, 1, recs, blocks=blk), 1)
    assert found > 0


def test_inter_dc_only_redecision(mats, sim):
    """inter DC-only blocks take the trellis's last_non_zero == 0 branch, which may drop the block (-1) and writes its own coded_score"""
    chk = M.checker()
    for fmt in (M.FMT_MPEG1, M.FMT_H263):
        st = M.make_state(mats, 0, fmt, seed=70 + fmt)
        cur, rf, off, stride = M.planes(500, 13, kinds=("dc_only",))
        blk = M.spatial(cur, rf, off, stride)
        recs = M.records(500, 14, intra=0)
        want = chk.run(st, M.Vlc(5, tie=True), 1, recs, blk)
        assert (want[1] == -1).any() and (want[1] == 0).any()
        M.compare(fmt, want, *M.run_sim(sim, st, M.Vlc(5, tie=True), 1, recs, blocks=blk), 1,
                  skip=M.undefined_blocks(st, M.Vlc(5, tie=True), 1, recs, blk))


def test_alternate_scan_recompute_keeps_last_index(mats, sim):
    """encode_mb_internal recomputes block_last_index for a quantiser other than ff_dct_quantize_c under alternate_scan
    (mpegvideo_enc.c:2312-2325); on the batch call's output that recompute changes nothing"""
    st = M.make_state(mats, 0, M.FMT_MPEG1, alt=1, matrices="random", seed=80)
    scan = np.frombuffer(bytes(st.scantable), np.uint8)
    assert scan[1] != 1 or scan[2] != 8                     # not the zigzag
    cur, rf, off, stride = M.planes(600, 15)
    blk = M.spatial(cur, rf, off, stride)
    recs = M.records(600, 16)
    for trellis in (0, 1):
        levels, last, _ = M.run_sim(sim, st, M.Vlc(6), trellis, recs, blocks=blk)
        assert (last > 0).sum() > 100
        assert np.array_equal(M.alternate_scan_recompute(levels, last, scan), last)


def test_real_trellis_runs(ref, mats):
    """libmpvqref.so runs its own copies of the static quantisers (not the aborting stand-ins of libavref.so), and the trellis decides
    differently from the plain quantiser"""
    fns = [C.c_void_p() for _ in range(3)]
    ref.lib.ref_mpvq_impl.argtypes = [C.POINTER(C.c_void_p)] * 3
    ref.lib.ref_mpvq_impl(*[C.byref(f) for f in fns])
    lo, hi = _mapping(M.MPVQ_REF)
    assert all(lo <= f.value < hi for f in fns)
    st = M.make_state(mats, 0, M.FMT_MPEG1, seed=90)
    cur, rf, off, stride = M.planes(300, 17)
    blk = M.spatial(cur, rf, off, stride)
    recs = M.records(300, 18, lambda2=np.uint32(5000))
    plain = ref.run(st, M.Vlc(7), 0, recs, blk)
    trellis = ref.run(st, M.Vlc(7), 1, recs, blk)
    assert (plain[0] != trellis[0]).any(axis=1).sum() > 30
    assert (trellis[3] != M.SCORE_UNSET).sum() > 100 and (plain[3] == M.SCORE_UNSET).all()


def _mapping(path):
    real = os.path.realpath(path)
    lo, hi = None, None
    with open("/proc/self/maps") as f:
        for line in f:
            if line.rstrip().endswith(real):
                a, b = [int(x, 16) for x in line.split()[0].split("-")]
                lo = a if lo is None else min(lo, a)
                hi = b if hi is None else max(hi, b)
    return lo, hi


def test_inv_aanscales_derived_equals_reference(ref):
    from oracle import loader
    want, got = np.zeros(64, np.uint16), np.zeros(64, np.uint16)
    ref.lib.ref_mpvq_inv_aanscales(want.ctypes.data_as(C.c_void_p))
    loader.port().lib.orc_mpvq_inv_aanscales(got.ctypes.data_as(C.c_void_p))
    assert np.array_equal(want, got)


# ---- the slots and the hook ------------------------------------------------------------------------------------------------------------

class FakeEncoder:
    """the MpegEncContext fields the slots read and write, as numpy cells an FFMpvQuantView points into"""

    def __init__(self, st, vlc, nr):
        from libav_b200 import tables
        self.ints = np.zeros(16, np.int32)          # 0 mb_intra 1 y_dc 2 c_dc 3 aic 4 lambda2 5 ibias 6 nbias 7 esc 8 minq 9 maxq
        self.ints[:10] = [0, 8, 8, st.h263_aic, 0, st.intra_quant_bias, st.inter_quant_bias, st.ac_esc_length, st.min_qcoeff, st.max_qcoeff]
        self.qi = np.ctypeslib.as_array(st.q_intra_matrix).reshape(32, 64).copy()
        self.qn = np.ctypeslib.as_array(st.q_inter_matrix).reshape(32, 64).copy()
        self.qi_p, self.qn_p = C.c_void_p(self.qi.ctypes.data), C.c_void_p(self.qn.ctypes.data)
        self.im = np.array(list(st.intra_matrix), np.uint16)
        self.nm = np.array(list(st.inter_matrix), np.uint16)
        self.scan = np.array(list(st.scantable), np.uint8)
        self.vlc = vlc                              # the tables must outlive the slots, as a codec's static tables do
        self.vlc_p = (C.c_void_p * 4)(*[t.ctypes.data for t in vlc.t])
        self.nr = nr
        self.es_p = C.c_void_p(nr.sum.ctypes.data if nr else None)
        self.off_p = C.c_void_p(nr.offset.ctypes.data if nr else None)
        self.count = nr.count if nr else np.zeros(2, np.int32)
        self.coded = np.full(8, M.SCORE_UNSET, np.int32)
        self.fns = (C.c_void_p * 2)()
        self.key = np.zeros(8, np.uint8)
        v = tables.FFMpvQuantView()
        cell = lambda k: self.ints.ctypes.data + 4 * k
        (v.mb_intra, v.y_dc_scale, v.c_dc_scale, v.h263_aic, v.lambda2, v.intra_quant_bias, v.inter_quant_bias, v.ac_esc_length,
         v.min_qcoeff, v.max_qcoeff) = [cell(k) for k in range(10)]
        v.q_intra_matrix, v.q_inter_matrix = C.addressof(self.qi_p), C.addressof(self.qn_p)
        v.intra_matrix, v.inter_matrix, v.scantable = self.im.ctypes.data, self.nm.ctypes.data, self.scan.ctypes.data
        base = C.addressof(self.vlc_p)
        v.intra_ac_vlc_length, v.intra_ac_vlc_last_length, v.inter_ac_vlc_length, v.inter_ac_vlc_last_length = [base + 8 * k for k in range(4)]
        v.dct_error_sum, v.dct_offset, v.dct_count, v.coded_score = C.addressof(self.es_p), C.addressof(self.off_p), self.count.ctypes.data, self.coded.ctypes.data
        v.dct_quantize, v.fast_dct_quantize = C.addressof(self.fns), C.addressof(self.fns) + 8
        v.fdct, v.out_format, v.mpeg_quant, v.idct_perm_none, v.quantizer_noise_shaping = st.fdct, st.out_format, st.mpeg_quant, 1, 0
        v.slice_context_count = 1
        self.view = v

    def slot(self, k):
        from libav_b200 import tables
        return C.cast(C.c_void_p(self.fns[k]), tables.DCT_QUANTIZE_FUNC)


def slot_cases(lib, mats, n=60):
    """the slots the hook installs, driven like encode_mb_internal drives s->dct_quantize (live fields change between calls), against the
    checker's dct_quantize on the same blocks in the same order: levels, return value, overflow, coded_score[n], the noise-reduction sums"""
    chk = M.checker()
    checked = 0
    for k, (label, st) in enumerate(M.states(mats)[::2]):
        vlc = M.Vlc(k)
        nr_slot, nr_ref = (M.NR(k), M.NR(k)) if k % 2 else (None, None)
        enc = FakeEncoder(st, vlc, nr_slot)
        key = C.c_void_p(enc.key.ctypes.data)
        for trellis in (0, 1):
            assert lib.ff_mpv_quantize_init_cuda(key, C.byref(enc.view), trellis) == 0, label
            assert enc.fns[1] and enc.fns[0] and (enc.fns[0] != enc.fns[1]) == bool(trellis)
            cur, rf, off, stride = M.planes(n, 40 + k)
            blk = M.spatial(cur, rf, off, stride)
            recs = M.records(n, 50 + k)
            skip = M.undefined_blocks(st, vlc, trellis, recs, blk, nr_ref)
            want = chk.run(st, vlc, trellis, recs, blk, nr_ref, post=False)
            for i in range(n):
                r = recs[i]
                bn = 4 if r["chroma"] else 0
                enc.ints[0], enc.ints[4] = r["intra"], r["lambda2"]
                enc.ints[2 if r["chroma"] else 1] = r["dc_scale"]
                enc.coded[bn] = M.SCORE_UNSET
                b = blk[i].copy()
                ovf = C.c_int(-1)
                last = enc.slot(0)(key, b.ctypes.data, bn, int(r["qscale"]), C.byref(ovf))
                if skip[i]:
                    continue
                assert (last, ovf.value, int(enc.coded[bn])) == (want[1][i], want[2][i], want[3][i]), (label, trellis, i)
                assert np.array_equal(b, want[0][i]), (label, trellis, i)
                checked += 1
            if nr_slot:
                assert np.array_equal(nr_slot.sum, nr_ref.sum) and np.array_equal(enc.count, nr_ref.count), label
        lib.ff_mpv_quantize_uninit_cuda(key)
    return checked


def hook_refusals(lib, mats):
    """refusals leave the context's two fields alone"""
    st = M.make_state(mats)
    enc = FakeEncoder(st, M.Vlc(1), None)
    key = C.c_void_p(enc.key.ctypes.data)
    for field, value in (("idct_perm_none", 0), ("fdct", 1), ("fdct", 3), ("quantizer_noise_shaping", 1), ("slice_context_count", 2),
                         ("slice_context_count", 8)):
        old = getattr(enc.view, field)
        setattr(enc.view, field, value)
        assert lib.ff_mpv_quantize_init_cuda(key, C.byref(enc.view), 1) == -1 and lib.avb200_last_error(), field
        assert not enc.fns[0] and not enc.fns[1], field
        setattr(enc.view, field, old)
    enc.view.scantable = None
    assert lib.ff_mpv_quantize_init_cuda(key, C.byref(enc.view), 0) == -1 and not enc.fns[0]
    lib.avb200_clear_error()                    # (the expected refusals leave their message pending)


def test_hostsim_slots(sim, mats):
    assert slot_cases(sim, mats) > 1000
    hook_refusals(sim, mats)


def batch_refusals(lib, upload, download, mats):
    """-1 with a message and every buffer as it was: a bad state (no handle at all), trellis on a state without VLC tables, misaligned
    blocks, NULL buffers; 0 blocks returns 0.  upload / download: host or device memory."""
    from libav_b200 import tables
    st = M.make_state(mats)
    for mutate in (lambda s: setattr(s, "fdct", 1), lambda s: setattr(s, "out_format", 4),
                   lambda s: s.scantable.__setitem__(5, s.scantable[6]), lambda s: (s.scantable.__setitem__(0, 1), s.scantable.__setitem__(1, 0))):
        b = tables.FFMpvQuantState.from_buffer_copy(st)
        mutate(b)
        lib.avb200_clear_error()
        assert not lib.ff_mpv_quant_state_cuda(C.byref(b), None) and lib.avb200_last_error()
    n = 37
    h_plain = lib.ff_mpv_quant_state_cuda(C.byref(st), None)
    assert h_plain
    rng = np.random.default_rng(1)
    blocks = rng.integers(-255, 256, (n + 1, 64)).astype(np.int16)
    recs = M.records(n, 2)
    last = np.full(n, 99, np.int32)
    d_blk, d_rec, d_last = upload(blocks), upload(recs), upload(last)
    base = d_blk
    for args, what in (((h_plain, 1, d_rec, None, None, None, None, 0, base, n, d_last, None, None, None), "trellis without VLC"),
                       ((h_plain, 0, d_rec, None, None, None, None, 0, base + 2, n, d_last, None, None, None), "misaligned blocks"),
                       ((h_plain, 0, d_rec, None, None, None, None, 0, base + 8, n, d_last, None, None, None), "misaligned blocks (8)"),
                       ((h_plain, 0, None, None, None, None, None, 0, base, n, d_last, None, None, None), "NULL recs"),
                       ((None, 0, d_rec, None, None, None, None, 0, base, n, d_last, None, None, None), "no state")):
        lib.avb200_clear_error()
        assert lib.ff_mpv_dct_quantize_batch_cuda(*args) == -1 and lib.avb200_last_error(), what
        assert np.array_equal(download(d_blk, blocks), blocks) and np.array_equal(download(d_last, last), last), what
    lib.avb200_clear_error()                    # (the expected refusals leave their message pending)
    assert lib.ff_mpv_dct_quantize_batch_cuda(h_plain, 0, d_rec, None, None, None, None, 0, base, 0, d_last, None, None, None) == 0
    assert np.array_equal(download(d_blk, blocks), blocks) and not lib.avb200_last_error()
    lib.ff_mpv_quant_state_free_cuda(h_plain)


def test_hostsim_batch_refusals(sim, mats):
    keep = []

    def upload(a):
        a = np.ascontiguousarray(a).copy()
        keep.append(a)
        return a.ctypes.data

    def download(p, like):
        return np.ctypeslib.as_array(C.cast(p, C.POINTER(C.c_uint8)), (like.nbytes,)).view(like.dtype).reshape(like.shape).copy()

    batch_refusals(sim, upload, download, mats)


def test_hook_follows_me_cmp_hook_in_reference_glue():
    """examples/reference_binding: ff_mpv_quantize_init_cuda comes after ff_me_cmp_enc_init_cuda, which must still see
    fast_dct_quantize == ff_dct_quantize_c, and gets avctx->trellis"""
    src = open(os.path.join(ROOT, "examples", "reference_binding", "dsp_init_cuda.c")).read()
    a = src.index("ff_me_cmp_enc_init_cuda(&s->mecc, s, &v)")
    b = src.index("ff_mpv_quantize_init_cuda(s, &q, s->avctx->trellis)")
    assert a < b
    assert ".slice_context_count = s->slice_context_count" in src[a:b]      # slice-threaded encoders are refused by the hook


ABI_PROBE = r"""
#include <stddef.h>
#include <stdio.h>
#include "avdsp_b200.h"
int main(void)
{
    printf("%zu %zu %zu %zu %zu %zu %zu %zu %zu %zu %zu %zu %zu\n", sizeof(FFMpvQuantState), offsetof(FFMpvQuantState, q_intra_matrix),
           offsetof(FFMpvQuantState, intra_matrix), offsetof(FFMpvQuantState, scantable), sizeof(FFMpvQuantRecord),
           offsetof(FFMpvQuantRecord, lambda2), sizeof(FFMpvNoiseReduction), sizeof(FFMpvQuantView), offsetof(FFMpvQuantView, dct_error_sum),
           offsetof(FFMpvQuantView, dct_quantize), offsetof(FFMpvQuantView, fdct), offsetof(FFMpvQuantView, quantizer_noise_shaping),
           offsetof(FFMpvQuantView, slice_context_count));
    return 0;
}
"""


def test_abi_of_the_new_structs(tmp_path):
    from libav_b200 import tables as T
    src = tmp_path / "probe.c"
    src.write_text(ABI_PROBE)
    exe = str(tmp_path / "probe")
    subprocess.run(["gcc", "-std=c99", "-Wall", "-Werror", "-I", os.path.join(ROOT, "include"), str(src), "-o", exe], check=True)
    got = [int(x) for x in subprocess.run([exe], check=True, capture_output=True, text=True).stdout.split()]
    want = [C.sizeof(T.FFMpvQuantState), T.FFMpvQuantState.q_intra_matrix.offset, T.FFMpvQuantState.intra_matrix.offset,
            T.FFMpvQuantState.scantable.offset, C.sizeof(T.FFMpvQuantRecord), T.FFMpvQuantRecord.lambda2.offset, C.sizeof(T.FFMpvNoiseReduction),
            C.sizeof(T.FFMpvQuantView), T.FFMpvQuantView.dct_error_sum.offset, T.FFMpvQuantView.dct_quantize.offset, T.FFMpvQuantView.fdct.offset,
            T.FFMpvQuantView.quantizer_noise_shaping.offset, T.FFMpvQuantView.slice_context_count.offset]
    assert got == want
    assert C.sizeof(T.FFMpvQuantRecord) == M.REC.itemsize == 8
