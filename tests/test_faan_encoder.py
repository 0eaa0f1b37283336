"""The encoder paths behind the FAAN forward DCT (fdct 6 = ff_faandct, FF_DCT_FAAN): the quantiser (FFMpvQuantState / FFMpvQuantView) and
the quant_psnr / bit / rd metrics (FFMECmpEncState / FFMECmpEncView), host-compiled and on the GPU, against the reference's own
mpegvideo_enc.c and me_cmp.c on contexts whose s->fdsp.fdct is ff_faandct (oracle/_ref/libfaanqref.so, libfaanencref.so: faan.mk).

The states are the existing suites' islow states with fdct 6: ff_convert_matrix treats ff_faandct like the islow transform
(mpegvideo_enc.c:95-99), so their q matrices are the FAAN encoder's.  Left out: the quantiser states with tiny matrices, whose trellis scores
wrap past 2^31 and read table entries the reference never writes (the suites find those blocks with the port, which has no FAAN transform),
and the metrics of the H.263 family, where the reference asserts on blocks that quantise to nothing (found with the port likewise)."""
import ctypes as C
import os

import numpy as np
import pytest

import enc_cases
import hostsim_build
import mpv_quant_cases as M
import test_mpv_quant_cpu as QCPU

FAAN = 6


def _ref_path(name):
    return os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "oracle", "_ref", name)


@pytest.fixture(scope="session")
def qref(built):
    if not os.path.exists(_ref_path("libfaanqref.so")):
        pytest.skip("oracle/_ref not built (no reference tree in this environment)")
    return M.Oracle(C.CDLL(_ref_path("libfaanqref.so")).ref_faanq_batch, "ref_faan")


class EncRef:
    """the FAAN encoder's quant_psnr / bit / rd and q matrices, with the interface enc_cases expects of a checker"""

    def __init__(self):
        lib = C.CDLL(_ref_path("libfaanencref.so"))
        self.me_cmp_quant = lib.ref_faanenc_me_cmp_quant
        self.me_cmp_quant.restype = C.c_int
        self.me_cmp_quant.argtypes = [C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_ssize_t, C.c_int, C.c_void_p]
        self.enc_qmatrices = lib.ref_faanenc_qmatrices
        self.enc_qmatrices.restype = None
        self.enc_qmatrices.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]


@pytest.fixture(scope="session")
def eref(built):
    if not os.path.exists(_ref_path("libfaanencref.so")):
        pytest.skip("oracle/_ref not built (no reference tree in this environment)")
    return EncRef()


@pytest.fixture(scope="session")
def mats(built):
    return M.matrices_checker()


def faan_states(mats):
    out = []
    for label, st in M.states(mats):
        if st.fdct == 0 and not label.endswith("_v2"):          # islow q matrices; v2 = the tiny matrices
            st.fdct = FAAN
            out.append((label.replace("fdct0", "faan"), st))
    assert len(out) == 8
    return out


@pytest.fixture
def faan_quant(monkeypatch, mats, qref):
    """the quantiser suites' case generators with FAAN states and the FAAN reference as checker"""
    st = faan_states(mats)
    monkeypatch.setattr(M, "states", lambda checker: st)
    monkeypatch.setattr(M, "checker", lambda: qref)
    monkeypatch.setattr(M, "undefined_blocks", lambda st, vlc, trellis, recs, blocks, nr=None: np.zeros(len(recs), bool))
    return qref


_ENC_STATES = enc_cases.states


def enc_faan_states(T):
    out = []
    for label, st in _ENC_STATES(T):
        if st.fdct_sel == 0 and st.dequant != 3:
            st.fdct_sel = FAAN
            out.append((label.replace("fdct0", "faan"), st))
    return out


def _quant_cases(mats, run, n, seed):
    """plain and trellis quantiser, noise reduction on and off, clip and elimination (post), every record shape of the suites"""
    checked = 0
    for label, st, vlc, trellis, recs, blk, nr in QCPU._cases(mats, n=n, seed=seed):
        nr1, nr2 = (nr.copy(), nr.copy()) if nr else (None, None)
        want = M.checker().run(st, vlc, trellis, recs, blk, nr1)
        M.compare(label, want, *run(st, vlc, trellis, recs, blk, nr2), trellis)
        if nr:
            assert np.array_equal(nr1.sum, nr2.sum) and np.array_equal(nr1.count, nr2.count), label
        checked += len(recs)
    return checked


# ---------------------------------------------------------------------------------------------------------------------------- CPU

def test_state_and_view_take_fdct_6_and_still_refuse_1_and_3(built, mats):
    sim = hostsim_build.fresh()
    st = faan_states(mats)[0][1]
    h = sim.ff_mpv_quant_state_cuda(C.byref(st), None)
    assert h, sim.avb200_last_error()
    sim.ff_mpv_quant_state_free_cuda(h)
    for bad in (1, 3, 7):
        st.fdct = bad
        assert not sim.ff_mpv_quant_state_cuda(C.byref(st), None)
        sim.avb200_clear_error()


def test_hostsim_quantiser_with_faan(faan_quant, mats):
    sim = hostsim_build.fresh()
    run = lambda st, vlc, trellis, recs, blk, nr: M.run_sim(sim, st, vlc, trellis, recs, blocks=blk, nr=nr)
    assert _quant_cases(mats, run, 300, 0) > 4000


def test_hostsim_quantiser_fused_front_end_with_faan(faan_quant, mats):
    """the kernel's own get_pixels / diff_pixels + FAAN transform equals the staged blocks, and the reference"""
    sim = hostsim_build.fresh()
    for k, (label, st) in enumerate(M.states(mats)):
        cur, rf, off, stride = M.planes(200, 40 + k)
        recs, vlc = M.records(200, 50 + k), M.Vlc(k)
        for trellis in (0, 1):
            blk = M.spatial(cur, rf, off, stride, inter=True)
            want = faan_quant.run(st, vlc, trellis, recs, blk)
            got = M.run_sim(sim, st, vlc, trellis, recs, pix=(cur, rf, off, stride))
            M.compare(label, want, *got, trellis)


def test_hostsim_quantiser_slots_with_faan(faan_quant, mats):
    sim = hostsim_build.fresh()
    assert QCPU.slot_cases(sim, mats) > 300


def _enc_protos(lib):
    from libav_b200 import _lib
    for name in ("ff_me_cmp_enc_state_cuda", "ff_me_cmp_enc_state_free_cuda", "ff_me_cmp_enc_batch_cuda", "ff_me_cmp_enc_init_cuda"):
        if name in _lib.PROTOTYPES and hasattr(lib, name):
            getattr(lib, name).restype, getattr(lib, name).argtypes = _lib.PROTOTYPES[name]


def test_hostsim_me_cmp_enc_with_faan(monkeypatch, eref):
    """quant_psnr / bit / rd (kinds 14-16), batch and slots, with state / view fdct 6"""
    sim = hostsim_build.fresh()
    _enc_protos(sim)
    monkeypatch.setattr(enc_cases, "states", enc_faan_states)

    def run_batch(kind, sidx, handle, cur, ref, recs, h):
        out, last = np.zeros(len(recs), np.int32), np.zeros(len(recs), np.int32)
        assert sim.ff_me_cmp_enc_batch_cuda(kind, sidx, handle, cur.ctypes.data, ref.ctypes.data, cur.strides[0], h, recs.ctypes.data, len(recs),
                                            out.ctypes.data, last.ctypes.data, None) == 0
        return out, last
    assert enc_cases.batch_cases(sim, run_batch, eref, None, n=12) > 2000
    assert enc_cases.slot_cases(sim, eref, None) > 200
    sim.avb200_clear_error()


# ---------------------------------------------------------------------------------------------------------------------------- GPU

@pytest.mark.gpu
def test_gpu_quantiser_with_faan(gpu, faan_quant, mats):
    import test_gpu_mpv_quant as G
    run = lambda st, vlc, trellis, recs, blk, nr: G.run_gpu(gpu, st, vlc, trellis, recs, blocks=blk, nr=nr)
    assert _quant_cases(mats, run, 2000, 3) > 30000


@pytest.mark.gpu
def test_gpu_quantiser_fused_front_end_with_faan(gpu, faan_quant, mats):
    import test_gpu_mpv_quant as G
    for k, (label, st) in enumerate(M.states(mats)):
        cur, rf, off, stride = M.planes(4000, 60 + k)
        recs, vlc = M.records(4000, 70 + k), M.Vlc(k)
        for trellis in (0, 1):
            for inter in (False, True):
                blk = M.spatial(cur, rf, off, stride, inter=inter)
                want = faan_quant.run(st, vlc, trellis, recs, blk)
                M.compare(label, want, *G.run_gpu(gpu, st, vlc, trellis, recs, pix=(cur, rf if inter else None, off, stride)), trellis)


@pytest.mark.gpu
def test_gpu_quantiser_slots_with_faan(gpu, faan_quant, mats):
    assert QCPU.slot_cases(gpu.lib, mats) > 300


@pytest.mark.gpu
def test_gpu_me_cmp_enc_with_faan(gpu, monkeypatch, eref):
    from libav_b200 import device
    monkeypatch.setattr(enc_cases, "states", enc_faan_states)

    def run_batch(kind, sidx, handle, cur, ref, recs, h):
        d_c, d_r, d_rec = device.DevBuf.from_numpy(cur), device.DevBuf.from_numpy(ref), device.DevBuf.from_numpy(recs)
        d_o, d_l = device.DevBuf(4 * len(recs)), device.DevBuf(4 * len(recs))
        gpu.check(gpu.lib.ff_me_cmp_enc_batch_cuda(kind, sidx, handle, d_c.ptr, d_r.ptr, cur.strides[0], h, d_rec.ptr, len(recs), d_o.ptr, d_l.ptr, None))
        device.sync()
        return d_o.download(np.int32, (len(recs),)), d_l.download(np.int32, (len(recs),))
    assert enc_cases.batch_cases(gpu.lib, run_batch, eref, None, n=24) > 4000
    assert enc_cases.slot_cases(gpu.lib, eref, None) > 200
    gpu.lib.avb200_clear_error()                                   # (slot_cases ends with a refusal it expects)
