"""GPU: H.263 overlapped block motion compensation through ff_mpv_motion_batch_cuda and the flush, byte for byte against the checker -- the
reference's apply_obmc (oracle/_ref/libmpvobmcref.so) where it travelled, else the plain-C port (oracle/port/orc_mpvobmc.c), which the
CPU suite pins to it.  CIF pictures of both roundings and all three size kinds, three per call; tiny pictures with edge vectors,
intra and stale neighbours; B pictures ignoring obmc; refusals; and an Annex F + Annex J flush: OBMC, residual, loop filter."""
import ctypes as C

import numpy as np
import pytest

import h263_cases as H
import mpv_mc_cases as M
import mpv_obmc_cases as O

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def ob_check(built):
    return O.checker_lib()


class GpuObmc(M.GpuPictures):
    def __init__(self, pics, obmc=True):
        from libav_b200 import device
        super().__init__(pics)
        self.obs = [device.DevBuf.from_numpy(np.ascontiguousarray(p.obmc)) if len(p.obmc) else None for p in pics]
        for i, p in enumerate(pics):
            self.arr[i].obmc = int(obmc)
            self.arr[i].obmc_recs = self.obs[i].ptr if self.obs[i] else None


def run_gpu(gpu, pics):
    from libav_b200 import device
    g = GpuObmc(pics)
    gpu.check(gpu.lib.ff_mpv_motion_batch_cuda(C.cast(g.arr, C.c_void_p), len(pics), g.rej.ptr, None), "ff_mpv_motion_batch_cuda")
    device.sync()
    return g.download(), g.rejected()


@pytest.mark.parametrize("no_rnd", [0, 1])
@pytest.mark.parametrize("ragged", [0, 1, 2])
def test_obmc_pictures(gpu, ob_check, no_rnd, ragged):
    pics = [O.obmc_picture(np.random.default_rng(10 * s + no_rnd + 3 * ragged), 22, 18, no_rnd=no_rnd, ragged=ragged, stale=0.3) for s in range(3)]
    got, rej = run_gpu(gpu, pics)
    assert rej == 0
    for i, pic in enumerate(pics):
        d = M.first_diff(got[i], O.run_ref(ob_check, pic))
        assert d is None, (i, d)


def test_edges_intra_stale_and_tiny(gpu, ob_check):
    pics = []
    for seed in range(24):
        rng = np.random.default_rng(seed)
        pics.append(O.obmc_picture(rng, int(rng.integers(1, 5)), int(rng.integers(1, 4)), no_rnd=seed & 1, ragged=seed % 3, intra=0.5,
                                   stale=0.6, far=0.3, edge=0.6))
    got, rej = run_gpu(gpu, pics)
    assert rej == 0
    for i, pic in enumerate(pics):
        assert M.first_diff(got[i], O.run_ref(ob_check, pic)) is None, i


def test_b_pictures_ignore_obmc(gpu):
    pic = O.obmc_picture(np.random.default_rng(9), 12, 8, b=1)
    got, rej = run_gpu(gpu, [pic])
    assert rej == 0 and M.first_diff(got[0], M.run_ref(M.checker_lib(), pic)) is None


def test_refusals_change_nothing(gpu):
    from libav_b200 import device
    pic = O.obmc_picture(np.random.default_rng(3), 6, 4)
    g = GpuObmc([pic])
    for field, value in [("quarter_sample", 1), ("out_format", 0), ("obmc_recs", None)]:
        old = getattr(g.arr[0], field)
        setattr(g.arr[0], field, value)
        assert gpu.lib.ff_mpv_motion_batch_cuda(C.cast(g.arr, C.c_void_p), 1, g.rej.ptr, None) == -1
        assert "OBMC" in gpu.last_error()
        gpu.lib.avb200_clear_error()
        setattr(g.arr[0], field, old)
    device.sync()
    assert all(np.array_equal(a, b) for a, b in zip(g.download()[0], pic.frame)) and g.rejected() == 0


def test_annex_f_and_j_flush(gpu, checker, ob_check):
    """OBMC P pictures, the residual a decoder records, then the loop filter -- against the reference OBMC, the IDCT / dequantiser oracles
    and the serial loop filter, in that order"""
    from libav_b200 import device, tables
    pics = [O.obmc_picture(np.random.default_rng(40 + i), 22, 18, no_rnd=i & 1, ragged=2 * (i == 2)) for i in range(3)]
    full = [(p.recs.copy(), p.obmc.copy()) for p in pics]
    batches = M.decoder_residual(checker, pics, np.random.default_rng(6), intra_share=0.1, xvid=False)
    for p, (recs0, ob0) in zip(pics, full):          # decoder_residual drops the intra macroblocks' records: keep the OBMC ones in step
        pos = {(int(r["mb_x"]), int(r["mb_y"])): k for k, r in enumerate(recs0)}
        p.obmc = np.ascontiguousarray(ob0[[pos[(int(r["mb_x"]), int(r["mb_y"]))] for r in p.recs]])
    want = [O.run_ref(ob_check, p) for p in pics]
    M.apply_residual(checker, M.xvid_checker(), want, batches)
    lf_check = H.checker_lib()
    rng = np.random.default_rng(7)
    tabs = [H.LfPicture(rng, 22, 18, skip=0.2, extra_cols=0) for _ in pics]
    for pic, w, t in zip(pics, want, tabs):
        prm = np.array([pic.p["linesize"], pic.p["uvlinesize"], 22, 18, t.mb_stride], np.int32)
        ct = np.ascontiguousarray(t.chroma, np.uint8)
        assert lf_check.picture((C.c_void_p * 3)(*[a.ctypes.data for a in w]), prm.ctypes.data, t.mb_type.ctypes.data, t.qscale.ctypes.data,
                                ct.ctypes.data) == 0
    g = GpuObmc(pics)
    res = M.GpuResidual(g, batches)
    dev = lambda a: device.DevBuf.from_numpy(np.ascontiguousarray(a))
    keep = [(dev(t.mb_type), dev(t.qscale)) for t in tabs]
    lf = (tables.FFH263LoopFilterPicture * len(pics))()
    for i, (pic, t) in enumerate(zip(pics, tabs)):
        for k in range(3):
            lf[i].data[k] = g.frames[i][k].ptr
        lf[i].linesize, lf[i].uvlinesize, lf[i].mb_width, lf[i].mb_height, lf[i].mb_stride = pic.p["linesize"], pic.p["uvlinesize"], 22, 18, t.mb_stride
        lf[i].mb_type, lf[i].qscale_table = keep[i][0].ptr, keep[i][1].ptr
        lf[i].chroma_qscale_table[:] = list(range(32))
    w = res.work(g)
    w.loop_filter, w.n_loop_filter = C.cast(lf, C.c_void_p), len(pics)
    gpu.check(gpu.lib.ff_mpv_flush_pictures_cuda(C.byref(w), None), "ff_mpv_flush_pictures_cuda")
    device.sync()
    for i, got in enumerate(g.download()):
        assert M.first_diff(got, want[i]) is None, (i, M.first_diff(got, want[i]))
    assert g.rejected() == 0
