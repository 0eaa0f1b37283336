"""GPU: ff_mpv_motion_batch_cuda and the flush point ff_mpv_flush_pictures_cuda, byte for byte against the checker -- the reference's own
ff_mpv_motion (oracle/_ref/libmpvmcref.so) where it travelled, else its plain-C restatement (oracle/port/orc_mpvmc.c), which the CPU suite
pins to the reference.  Every scenario of the CPU suite at a larger size; sixteen stacked 1080p pictures in one call; records the
kernel does not take and records with extreme vectors and positions (counted, untouched, and run without a fault); pictures refused as a
whole (-1, nothing changed); the flush with the simple and the Xvid IDCT, plain and dequant-fused, frame and field DCT, the coefficient
arena checked where `clear` is set."""
import ctypes as C

import numpy as np
import pytest

import mpv_mc_cases as M
from test_mpv_mc_cpu import SCENARIOS, bad_records, scenario_picture

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="session")
def mc_check(built):
    """run(pic) -> the frame planes the checker reconstructs from the picture's accepted records"""
    lib = M.checker_lib()
    return lambda pic: M.run_ref(lib, pic)


def run_gpu(gpu, pics, stream=None):
    from libav_b200 import device
    g = M.GpuPictures(pics)
    gpu.check(gpu.lib.ff_mpv_motion_batch_cuda(C.cast(g.arr, C.c_void_p), len(pics), g.rej.ptr, stream), "ff_mpv_motion_batch_cuda")
    device.sync()
    return g.download(), g.rejected()


@pytest.mark.parametrize("name", list(SCENARIOS))
def test_scenarios(gpu, mc_check, name):
    pic = scenario_picture(name, 7 + len(name), mb_w=23, mb_h=14)
    got, rej = run_gpu(gpu, [pic])
    assert rej == 0
    d = M.first_diff(got[0], mc_check(pic))
    assert d is None, (name, d)


@pytest.mark.parametrize("fmt,structure,custom", [(0, M.FRAME, 0), (0, M.BOTTOM, 0), (2, M.FRAME, 0), (2, M.FRAME, 1)])
def test_every_type_near_edges(gpu, mc_check, fmt, structure, custom):
    for t in M.mv_types(fmt, structure):
        for qpel in ((0, 1) if fmt == 2 else (0,)):
            rng = np.random.default_rng(31 + t)
            pic = M.Picture(rng, fmt, 4, 4, structure=structure, first_field=t & 1, b=qpel, no_rnd=1 - qpel, qpel=qpel,
                            width=61 if fmt == 2 else None, height=53 if fmt == 2 else None, custom_edges=bool(custom))
            M.make_records(rng, pic, far=0.3, edge=0.6, types=[t])
            got, rej = run_gpu(gpu, [pic])
            assert rej == 0 and M.first_diff(got[0], mc_check(pic)) is None, (t, qpel, M.first_diff(got[0], mc_check(pic)))


def test_tiny_pictures(gpu, mc_check):
    """pictures narrower / shorter than 16 samples: the direct read one column / row past the aligned plane"""
    pics = []
    for seed in range(16):
        rng = np.random.default_rng(seed)
        pic = M.Picture(rng, 2, 1, 1, no_rnd=seed & 1, qpel=seed >> 3, width=int(rng.integers(2, 16)), height=int(rng.integers(2, 16)))
        pic.recs = np.zeros(1, M.REC)
        pic.recs[0]["mv_dir"] = 1
        pic.recs[0]["mv"][0, 0] = rng.integers(0, 4, 2)
        pics.append(pic)
    got, rej = run_gpu(gpu, pics)
    assert rej == 0
    for i, pic in enumerate(pics):
        assert M.first_diff(got[i], mc_check(pic)) is None, i


def test_sixteen_stacked_1080p_pictures(gpu, mc_check):
    """one call, sixteen 1920x1088 pictures of both families: MPEG-2 frame / field, P / B; MPEG-4 quarter-sample 4MV B pictures"""
    names = ["mpeg2_frame_p", "mpeg2_frame_b", "mpeg2_top_first_p", "mpeg2_bottom_first_b", "mpeg4_qpel_b_ragged", "mpeg4_qpel_p_ragged",
             "mpeg2_frame_b", "mpeg4_hpel_b_ragged"] * 2
    pics = [scenario_picture(n, 500 + i, mb_w=120, mb_h=68) for i, n in enumerate(names)]
    got, rej = run_gpu(gpu, pics)
    assert rej == 0
    for i, pic in enumerate(pics):
        d = M.first_diff(got[i], mc_check(pic))
        assert d is None, (i, names[i], d)


@pytest.mark.parametrize("name", ["mpeg2_frame_b", "mpeg2_top_second_p", "mpeg4_qpel_b_ragged", "h263_hpel_p"])
def test_rejected_and_extreme_records(gpu, mc_check, name):
    """a third of the records outside the picture or of an unknown / foreign type, the rest with vectors mostly at the int16 extremes:
    a normal run, the rejected ones counted and their macroblocks untouched"""
    rng = np.random.default_rng(9)
    pic = scenario_picture(name, 19, mb_w=17, mb_h=10)
    M.make_records(rng, pic, far=0.8, edge=0.2)
    pic.recs = bad_records(pic, rng)
    n_bad = int((~pic.accepted()).sum())
    got, rej = run_gpu(gpu, [pic])
    assert rej == n_bad > 0
    assert M.first_diff(got[0], mc_check(pic)) is None


def test_picture_refusal_changes_nothing(gpu):
    from libav_b200 import device
    pic = scenario_picture("mpeg4_qpel_p_ragged", 3, mb_w=9, mb_h=5)
    g = M.GpuPictures([pic])
    for field, value in [("obmc", 1), ("sprite", 1), ("chroma_format", 2), ("out_format", 1), ("lowres", 1)]:
        old = getattr(g.arr[0], field)
        setattr(g.arr[0], field, value)
        assert gpu.lib.ff_mpv_motion_batch_cuda(C.cast(g.arr, C.c_void_p), 1, g.rej.ptr, None) == -1
        assert gpu.last_error()
        gpu.lib.avb200_clear_error()
        setattr(g.arr[0], field, old)
    device.sync()
    got = g.download()[0]
    assert all(np.array_equal(a, b) for a, b in zip(got, pic.frame)) and g.rejected() == 0


# ------------------------------------------------------------------------------------------------------------------------------- flush

def run_flush(gpu, checker, mc_check, pics, batches):
    """the flush on the device against the chained checker (reference MC, then the residual batches through the IDCT / inverse quantiser
    oracles in the same order); the coefficient arenas of `clear` batches are compared too"""
    from libav_b200 import device
    want = [mc_check(p) for p in pics]
    keeps = M.apply_residual(checker, M.xvid_checker(), want, batches)
    g = M.GpuPictures(pics)
    res = M.GpuResidual(g, batches)
    w = res.work(g)
    gpu.check(gpu.lib.ff_mpv_flush_pictures_cuda(C.byref(w), None), "ff_mpv_flush_pictures_cuda")
    device.sync()
    got = g.download()
    for pi in range(len(pics)):
        d = M.first_diff(got[pi], want[pi])
        assert d is None, (pi, d)
    for b, d_b, keep in zip(batches, res.blocks, keeps):
        if b["clear"]:
            after = d_b.download(np.int16, b["blocks"].shape)
            assert not after[keep].any() and np.array_equal(after[~keep], b["blocks"][~keep])
    assert g.rejected() == 0


def test_flush_point(gpu, checker, mc_check):
    """MC of two pictures, then residual batches through every kind of entry point: simple and Xvid, plain put / add and dequant-fused
    (intra and inter kinds), frame and field DCT, with and without clear"""
    pics = [scenario_picture("mpeg2_frame_b", 61, mb_w=30, mb_h=17), scenario_picture("mpeg4_qpel_p_ragged", 62, mb_w=22, mb_h=18)]
    rng = np.random.default_rng(4)
    # (picture, plane, transform, dequant, mode, field_dct, clear)
    plan = [(0, 0, 0, -1, 1, 0, 1), (0, 0, 0, 4, 1, 1, 0), (0, 1, 0, 2, 0, 0, 1), (0, 2, 1, -1, 1, 0, 0),
            (1, 0, 1, 6, 1, 1, 1), (1, 0, 1, -1, 1, 0, 1), (1, 1, 1, 5, 0, 0, 0), (1, 2, 0, 1, 1, 0, 1), (1, 0, 0, 3, 0, 0, 1)]
    mbs = {0: [(x, y) for y in range(17) for x in range(30)], 1: [(x, y) for y in range(18) for x in range(22)]}
    for k in mbs:
        rng.shuffle(mbs[k])
    used, batches = {}, []
    for i, (pi, pl, tr, dq, mode, fd, clear) in enumerate(plan):
        pic = pics[pi]
        start = used.get((pi, pl), 0)
        used[(pi, pl)] = start + 60
        ls = pic.p["linesize"] if pl == 0 else pic.p["uvlinesize"]
        offs = []
        for x, y in mbs[pi][start:start + 60]:
            if pl == 0:
                o, lower = 16 * y * ls + 16 * x, ls if fd else 8 * ls
                offs += [o, o + 8, o + lower, o + lower + 8]
            else:
                offs.append(8 * y * ls + 8 * x)
        stride = 2 * ls if (fd and pl == 0) else ls
        batches.append(M.residual_batch(checker, pics, pi, pl, tr, dq, mode, offs, stride, clear, 90 + i, i & 1, (i >> 1) & 1))
    run_flush(gpu, checker, mc_check, pics, batches)


def test_flush_decoder_shaped(gpu, checker, mc_check):
    """the residual a decoder records (tests/mpv_mc_cases.py decoder_residual): intra macroblocks without MC, coded inter blocks, frame and
    field DCT in frame pictures, field pictures of both parities, MPEG-4 with the Xvid IDCT"""
    names = ["mpeg2_frame_b", "mpeg2_top_first_p", "mpeg2_bottom_second_p", "mpeg4_qpel_b_ragged", "h263_custom_size_hpel_p"]
    pics = [scenario_picture(n, 70 + i, mb_w=20, mb_h=12) for i, n in enumerate(names)]
    batches = M.decoder_residual(checker, pics, np.random.default_rng(5), intra_share=0.15, xvid=True)
    run_flush(gpu, checker, mc_check, pics, batches)


def test_flush_refuses_a_bad_batch_before_launching(gpu):
    from libav_b200 import device, tables
    pic = scenario_picture("mpeg2_frame_p", 5, mb_w=6, mb_h=4)
    g = M.GpuPictures([pic])
    b = tables.FFMpvResidualBatch()
    b.transform, b.dequant, b.mode, b.n = 2, -1, 1, 1
    w = tables.FFMpvPictureWork()
    w.pictures, w.n_pictures, w.rejected = C.cast(g.arr, C.c_void_p), 1, g.rej.ptr
    w.residual, w.n_residual = C.cast(C.pointer(b), C.c_void_p), 1
    assert gpu.lib.ff_mpv_flush_pictures_cuda(C.byref(w), None) == -1
    assert "residual" in gpu.last_error()
    gpu.lib.avb200_clear_error()
    device.sync()
    assert all(np.array_equal(a, b) for a, b in zip(g.download()[0], pic.frame))
