"""GPU: the H.263 deblocking filter through the C ABI, byte for byte against the checker -- the reference's serial driver
(oracle/_ref/libh263ref.so) where it travelled, else the two-pass plain-C restatement (oracle/port/orc_h263.c), which the CPU suite pins
to it.  ff_h263_loop_filter_batch_cuda over the CPU suite's pictures; a stacked call of 16CIF (1408x1152) and CIF pictures with the
padding checked; refusals that change nothing; the H263DSPContext slots installed by ff_h263dsp_init_cuda, called with host pointers; and
a decoder-shaped flush -- motion compensation, intra / inter residual batches, then the loop filter -- against the chained checker."""
import ctypes as C

import numpy as np
import pytest

import h263_cases as H
import mpv_mc_cases as M
from test_h263_cpu import cases, refusal_cases, slot_sweep
from test_mpv_mc_cpu import scenario_picture

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def lf_check(built):
    return H.checker_lib()


def run_gpu(gpu, pics, stream=None):
    from libav_b200 import device
    g = H.GpuLf(pics)
    gpu.check(gpu.lib.ff_h263_loop_filter_batch_cuda(C.cast(g.arr, C.c_void_p), len(pics), stream), "ff_h263_loop_filter_batch_cuda")
    device.sync()
    return g.download()


@pytest.mark.parametrize("seed", [1, 2])
def test_cpu_suite_pictures(gpu, lf_check, seed):
    """every picture of the CPU suite (1 x N, N x 1, 1 x 1 and larger; skip shares 0 .. 1; both chroma tables), all in one call"""
    named = list(cases(seed))
    got = run_gpu(gpu, [p for _, p in named])
    for (name, pic), g in zip(named, got):
        d = H.first_diff(g, H.run_serial(lf_check, pic))
        assert d is None, (name, d)


def test_stacked_16cif_and_cif(gpu, lf_check):
    """one call of 4 16CIF and 14 CIF pictures (two launches), odd and aligned linesizes, both chroma tables"""
    rng = np.random.default_rng(17)
    pics = [H.LfPicture(rng, 88, 72, skip=[0.1, 0.5][i & 1], chroma=H.ANNEX_T_CHROMA_QSCALE if i & 1 else None, extra_cols=[64, 3][i & 1])
            for i in range(4)]
    pics += [H.LfPicture(rng, 22, 18, skip=float(rng.random()), chroma=H.ANNEX_T_CHROMA_QSCALE if i % 3 else None) for i in range(14)]
    got = run_gpu(gpu, pics)
    for i, (g, pic) in enumerate(zip(got, pics)):
        d = H.first_diff(g, H.run_serial(lf_check, pic))
        assert d is None, (i, d)


def test_on_a_stream(gpu, lf_check):
    import libav_b200._lib as L
    from libav_b200 import device
    rng = np.random.default_rng(2)
    pics = [H.LfPicture(rng, 30, 20, skip=0.2)]
    s = L.lib.avb200_stream_create()
    try:
        got = run_gpu(gpu, pics, s)
        L.check(L.lib.avb200_stream_sync(s), "stream sync")
    finally:
        L.lib.avb200_stream_destroy(s)
    device.sync()
    assert H.first_diff(got[0], H.run_serial(lf_check, pics[0])) is None


def test_refusals_change_nothing(gpu):
    from libav_b200 import device
    rng = np.random.default_rng(3)
    for name, mutate in list(refusal_cases(rng)) + [("shared frame", lambda arr: arr.__setitem__(1, arr[0]))]:
        pics = [H.LfPicture(rng, 6, 4, skip=0.0, extra_cols=0), H.LfPicture(rng, 3, 3, skip=0.0)]
        g = H.GpuLf(pics)
        mutate(g.arr)
        assert gpu.lib.ff_h263_loop_filter_batch_cuda(C.cast(g.arr, C.c_void_p), 2, None) == -1, name
        assert gpu.last_error(), name
        gpu.lib.avb200_clear_error()
        device.sync()
        assert all(np.array_equal(a, b) for got, p in zip(g.download(), pics) for a, b in zip(got, p.bufs)), name


def test_slots(gpu, lf_check):
    """the slots ff_h263dsp_init_cuda installs, with host buffers, against the checker's C functions: every qscale, every d range, both
    stride signs, the whole 12 x 12 buffer around the call compared"""
    from libav_b200 import tables
    t = tables.H263DSPContext()
    gpu.lib.ff_h263dsp_init_cuda(C.byref(t))
    if hasattr(lf_check, "ref_h263dsp_init"):
        r = tables.H263DSPContext()
        lf_check.ref_h263dsp_init(C.byref(r))
        want = lambda v, b, o, s, q: (r.h263_h_loop_filter if v else r.h263_v_loop_filter)(C.cast(b.ctypes.data + o, C.POINTER(C.c_uint8)), s, q)
    else:
        want = lambda v, b, o, s, q: (lf_check.h_loop_filter if v else lf_check.v_loop_filter)(b.ctypes.data + o, s, q)
    slot_sweep(lambda v, a, o, s, q: (t.h263_h_loop_filter if v else t.h263_v_loop_filter)(C.cast(a.ctypes.data + o, C.POINTER(C.c_uint8)), s, q),
               want)
    assert not gpu.last_error()


def test_decoder_flush_with_the_loop_filter(gpu, checker, lf_check):
    """H.263 P pictures (one of them a custom size): their motion compensation, the intra / inter residual a decoder records, then the
    loop filter over every picture -- against the reference MC, the IDCT / dequantiser oracles and the serial loop filter, in that order"""
    from libav_b200 import device, tables
    names = ["h263_hpel_p", "h263_hpel_p_no_rounding", "h263_custom_size_hpel_p"]
    pics = [scenario_picture(n, 90 + i, mb_w=22, mb_h=18) for i, n in enumerate(names)]
    batches = M.decoder_residual(checker, pics, np.random.default_rng(6), intra_share=0.15, xvid=False)
    rng = np.random.default_rng(7)
    tabs = [H.LfPicture(rng, 22, 18, skip=0.25, chroma=H.ANNEX_T_CHROMA_QSCALE if i == 2 else None, extra_cols=0) for i in range(len(pics))]
    mc_lib = M.checker_lib()
    want = [M.run_ref(mc_lib, p) for p in pics]
    M.apply_residual(checker, M.xvid_checker(), want, batches)
    for pic, w, t in zip(pics, want, tabs):
        prm = np.array([pic.p["linesize"], pic.p["uvlinesize"], 22, 18, t.mb_stride], np.int32)
        ct = np.ascontiguousarray(t.chroma, np.uint8)
        assert lf_check.picture((C.c_void_p * 3)(*[a.ctypes.data for a in w]), prm.ctypes.data, t.mb_type.ctypes.data, t.qscale.ctypes.data,
                                ct.ctypes.data) == 0
    g = M.GpuPictures(pics)
    res = M.GpuResidual(g, batches)
    dev = lambda a: device.DevBuf.from_numpy(np.ascontiguousarray(a))
    keep = [(dev(t.mb_type), dev(t.qscale)) for t in tabs]
    lf = (tables.FFH263LoopFilterPicture * len(pics))()
    for i, (pic, t) in enumerate(zip(pics, tabs)):
        for k in range(3):
            lf[i].data[k] = g.frames[i][k].ptr
        lf[i].linesize, lf[i].uvlinesize, lf[i].mb_width, lf[i].mb_height, lf[i].mb_stride = pic.p["linesize"], pic.p["uvlinesize"], 22, 18, t.mb_stride
        lf[i].mb_type, lf[i].qscale_table = keep[i][0].ptr, keep[i][1].ptr
        lf[i].chroma_qscale_table[:] = [int(x) for x in t.chroma]
    w = res.work(g)
    w.loop_filter, w.n_loop_filter = C.cast(lf, C.c_void_p), len(pics)
    gpu.check(gpu.lib.ff_mpv_flush_pictures_cuda(C.byref(w), None), "ff_mpv_flush_pictures_cuda")
    device.sync()
    for i, got in enumerate(g.download()):
        d = M.first_diff(got, want[i])
        assert d is None, (names[i], d)
    assert g.rejected() == 0
