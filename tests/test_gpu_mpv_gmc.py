"""GPU: MPEG-4 global motion compensation (S-VOPs) through ff_mpv_motion_batch_cuda and the flush, and the MpegVideoDSPContext slots, byte
for byte against the checker -- the reference's ff_mpv_motion on S-VOPs and gmc1_c / ff_gmc_c (oracle/_ref) where they travelled, else
the plain-C port (oracle/port/orc_mpvgmc.c), which the CPU suite pins to them.  1, 2 and 3 warping points at every accuracy, both
roundings, half- and quarter-sample; hand-set parameters on tiny and ragged pictures; stacked 720x576 and 1920x1088 S-VOPs; S, P and B
pictures in one call; refusals; an S-VOP flush with the Xvid residual; the slots with host buffers."""
import ctypes as C

import numpy as np
import pytest

import mpv_gmc_cases as G
import mpv_mc_cases as M

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def g_check(built):
    return G.checker_lib()


def run_gpu(gpu, pics):
    from libav_b200 import device
    g = G.GpuSvops(pics)
    gpu.check(gpu.lib.ff_mpv_motion_batch_cuda(C.cast(g.arr, C.c_void_p), len(pics), g.rej.ptr, None), "ff_mpv_motion_batch_cuda")
    device.sync()
    return g.download(), g.rejected()


def _svop(seed, mb_w, mb_h, pts, acc, no_rnd=0, qpel=0, ragged=True, **kw):
    rng = np.random.default_rng(seed)
    pic = G.svop(rng, mb_w, mb_h, params=(0, 1, [[0, 0], [0, 0]], [[2, 0], [0, 2]]), no_rnd=no_rnd, qpel=qpel, ragged=ragged, **kw)
    p = pic.p
    pic.sprite = G.random_params(rng, p["width"], p["height"], mb_w, mb_h, p["h_edge_pos"], p["v_edge_pos"], pts=pts, acc=acc)
    return pic


@pytest.mark.parametrize("pts", [1, 2, 3])
@pytest.mark.parametrize("no_rnd", [0, 1])
def test_svops(gpu, g_check, pts, no_rnd):
    pics = [_svop(100 * pts + 10 * no_rnd + acc, 22, 18, pts, acc, no_rnd, qpel=acc & 1, ragged=acc >= 2) for acc in range(4)]
    got, rej = run_gpu(gpu, pics)
    assert rej == 0
    for i, pic in enumerate(pics):
        d = M.first_diff(got[i], G.run_ref(g_check, pic))
        assert d is None, (i, pic.sprite, d)


@pytest.mark.parametrize("kind", ["clamp", "edge1", "hpel1"])
def test_raw_parameters_tiny_and_ragged(gpu, g_check, kind):
    pics = []
    for seed in range(24):
        rng = np.random.default_rng(500 + seed)
        mb_w, mb_h = (int(rng.integers(1, 3)), int(rng.integers(1, 3))) if seed % 3 == 0 else (6, 4)
        pic = G.svop(rng, mb_w, mb_h, params=(0, 1, [[0, 0], [0, 0]], [[2, 0], [0, 2]]), no_rnd=seed & 1, qpel=(seed >> 1) & 1,
                     ragged=seed % 2 == 0, mcsel=0.85, intra=0.05)
        pic.sprite = G.raw_params(rng, pic, kind, int(rng.integers(0, 4)))
        pics.append(pic)
    got, rej = run_gpu(gpu, pics)
    assert rej == 0
    for i, pic in enumerate(pics):
        assert M.first_diff(got[i], G.run_ref(g_check, pic)) is None, (i, pic.sprite)


@pytest.mark.parametrize("mb_w,mb_h", [(45, 36), (120, 68)])
def test_stacked_full_size_svops(gpu, g_check, mb_w, mb_h):
    """720x576 and 1920x1088 S-VOPs, 2- and 3-point warps and translations, mostly mcsel macroblocks"""
    pics = [_svop(900 + i + mb_w, mb_w, mb_h, 1 + i % 3, (i * 3) % 4, no_rnd=i & 1, qpel=(i >> 1) & 1, ragged=False, mcsel=0.7)
            for i in range(3)]
    got, rej = run_gpu(gpu, pics)
    assert rej == 0
    for i, pic in enumerate(pics):
        assert M.first_diff(got[i], G.run_ref(g_check, pic)) is None, (i, pic.sprite)


def test_mixed_s_p_b_call(gpu, g_check):
    """S-VOPs (more than one launch of them), P and B pictures in one call, each routed to its kernel"""
    pics = [_svop(40 + i, 3, 3, 1 + i % 3, i % 4, i & 1, (i >> 1) & 1) for i in range(18)]
    rng = np.random.default_rng(91)
    for b in (0, 1, 0):
        p = M.Picture(rng, 2, 5, 4, b=b, qpel=b)
        M.make_records(rng, p)
        pics.append(p)
    got, rej = run_gpu(gpu, pics)
    assert rej == 0
    for i, p in enumerate(pics):
        assert M.first_diff(got[i], G.run_ref(g_check, p)) is None, i


def test_refusals_change_nothing(gpu):
    from libav_b200 import device
    pic = _svop(3, 6, 4, 2, 2, ragged=False)
    g = G.GpuSvops([pic])
    for field, value in [("b_picture", 1), ("out_format", 0), ("real_sprite_warping_points", 0), ("sprite_warping_accuracy", 4)]:
        old = getattr(g.arr[0], field)
        setattr(g.arr[0], field, value)
        assert gpu.lib.ff_mpv_motion_batch_cuda(C.cast(g.arr, C.c_void_p), 1, g.rej.ptr, None) == -1
        assert "sprite" in gpu.last_error()
        gpu.lib.avb200_clear_error()
        setattr(g.arr[0], field, old)
    device.sync()
    assert all(np.array_equal(a, b) for a, b in zip(g.download()[0], pic.frame)) and g.rejected() == 0


def test_svop_flush_with_xvid_residual(gpu, checker, g_check):
    """S-VOPs through the flush: GMC motion compensation, then the Xvid-written residual (intra blocks put_dct with the h263_intra
    dequantiser fused, inter blocks add_dct) -- against the GMC checker and the IDCT / dequantiser oracles, in that order"""
    from libav_b200 import device
    pics = [_svop(60 + i, 22, 18, 1 + i, i, no_rnd=i & 1, qpel=i == 1, ragged=i == 2) for i in range(3)]
    batches = M.decoder_residual(checker, pics, np.random.default_rng(8), intra_share=0.08, xvid=True)
    want = [G.run_ref(g_check, p) for p in pics]
    M.apply_residual(checker, M.xvid_checker(), want, batches)
    g = G.GpuSvops(pics)
    res = M.GpuResidual(g, batches)
    w = res.work(g)
    gpu.check(gpu.lib.ff_mpv_flush_pictures_cuda(C.byref(w), None), "ff_mpv_flush_pictures_cuda")
    device.sync()
    for i, got in enumerate(g.download()):
        assert M.first_diff(got, want[i]) is None, (i, M.first_diff(got, want[i]))
    assert g.rejected() == 0


def test_slots_with_host_buffers(gpu):
    """the slots ff_mpegvideodsp_init_cuda installs, called with host pointers, against gmc1_c / ff_gmc_c (or the port)"""
    from libav_b200 import tables
    ours = tables.MpegVideoDSPContext()
    gpu.lib.ff_mpegvideodsp_init_cuda(C.byref(ours))
    ref = G.ref_lib()
    if ref is not None:
        theirs = tables.MpegVideoDSPContext()
        ref.ref_mpegvideodsp_init(C.byref(theirs))
        gmc1, gmc = theirs.gmc1, theirs.gmc
    else:
        port = G.port_lib()
        gmc1 = lambda d, s, *a: port.gmc1(C.cast(d, C.c_void_p), C.cast(s, C.c_void_p), *a)
        gmc = lambda d, s, *a: port.gmc(C.cast(d, C.c_void_p), C.cast(s, C.c_void_p), *a)
    u8 = lambda a, o=0: C.cast(a.ctypes.data + o, C.POINTER(C.c_uint8))
    rng = np.random.default_rng(13)
    stride = 40
    for it in range(200):
        h = (8, 16)[it & 1]
        src = rng.integers(0, 256, (h + 6, stride), dtype=np.uint8)
        dst = rng.integers(0, 256, (h + 2, stride), dtype=np.uint8)
        want = dst.copy()
        x16, y16, rounder = int(rng.integers(0, 16)), int(rng.integers(0, 16)), 127 + (it >> 1 & 1)
        ours.gmc1(u8(dst, 3), u8(src, stride + 5), stride, h, x16, y16, rounder)
        gmc1(u8(want, 3), u8(src, stride + 5), stride, h, x16, y16, rounder)
        assert np.array_equal(dst, want), ("gmc1", it)
        shift = 1 + it % 4
        one = 1 << (16 + shift)
        w, hh = int(rng.integers(2, 36)), int(rng.integers(2, h + 6))
        ox, oy = int(rng.integers(-10, w + 10)) * one + int(rng.integers(0, one)), int(rng.integers(-10, hh + 10)) * one + int(rng.integers(0, one))
        d = [int(one * rng.uniform(0.4, 1.6)), int(one * rng.uniform(-0.5, 0.5)), int(one * rng.uniform(-0.5, 0.5)), int(one * rng.uniform(0.4, 1.6))]
        if not all(G._fits(ox + d[0] * cx + d[1] * cy, oy + d[2] * cx + d[3] * cy) for cx in (0, 8) for cy in (0, h)):
            continue
        args = (stride, h, ox, oy, d[0], d[1], d[2], d[3], shift, int(rng.integers(0, 1 << (2 * shift))), w, hh)
        dst = rng.integers(0, 256, (h, stride), dtype=np.uint8)
        want = dst.copy()
        ours.gmc(u8(dst), u8(src), *args)
        gmc(u8(want), u8(src), *args)
        assert np.array_equal(dst, want), ("gmc", it, args)
