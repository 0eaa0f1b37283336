"""GPU: MPEG-2 4:2:2 / 4:4:4 and interlaced MPEG-4 pictures through ff_mpv_motion_batch_cuda and the flush point
ff_mpv_flush_pictures_cuda, byte for byte against the reference's own ff_mpv_motion (oracle/_ref/libmpvcfref.so, libmpvmcref.so,
libmpvgmcref.so) and, for the flush, the chained checker (that motion compensation, then the IDCT and inverse quantiser oracles).  The
residual path is unchanged: these flushes show that 4:2:2 field-DCT chroma, 4:4:4's twelve blocks and interlaced MPEG-4's field-DCT
luma go through it as they are."""
import ctypes as C

import numpy as np
import pytest

import mpv_ilace_cases as I
import mpv_mc_cases as M

pytestmark = [pytest.mark.gpu, pytest.mark.skipif(not I.have_reference(), reason="the reference was not built")]


def run_gpu(gpu, pics):
    from libav_b200 import device
    g = I.GpuPics(pics)
    gpu.check(gpu.lib.ff_mpv_motion_batch_cuda(C.cast(g.arr, C.c_void_p), len(pics), g.rej.ptr, None), "ff_mpv_motion_batch_cuda")
    device.sync()
    return g.download(), g.rejected()


def check(gpu, pics):
    got, rej = run_gpu(gpu, pics)
    assert rej == sum(int((~p.accepted()).sum()) for p in pics)
    for i, (g, p) in enumerate(zip(got, pics)):
        d = M.first_diff(g, I.run_ref(p))
        assert d is None, (i, d)


@pytest.mark.parametrize("cf", [2, 3])
@pytest.mark.parametrize("structure,first,b,no_rnd", [(M.FRAME, 1, 0, 1), (M.FRAME, 1, 1, 0), (M.TOP, 1, 0, 0), (M.BOTTOM, 0, 0, 0),
                                                     (M.TOP, 0, 1, 0)])
def test_chroma_format(gpu, cf, structure, first, b, no_rnd):
    rng = np.random.default_rng(500 + 50 * cf + 10 * structure + 4 * first + 2 * b + no_rnd)
    check(gpu, [I.cf_picture(rng, cf, 23, 14, structure=structure, first_field=first, b=b, no_rnd=no_rnd, far=0.15, edge=0.45)])


@pytest.mark.parametrize("qpel", [0, 1])
@pytest.mark.parametrize("bugs", [0, I.BUG_HPEL_CHROMA])
@pytest.mark.parametrize("b,no_rnd", [(0, 1), (1, 0)])
def test_interlaced_mpeg4(gpu, qpel, bugs, b, no_rnd):
    rng = np.random.default_rng(600 + 8 * qpel + 4 * (bugs != 0) + 2 * b + no_rnd)
    check(gpu, [I.ilace_picture(rng, 23, 14, b=b, qpel=qpel, bugs=bugs, no_rnd=no_rnd, ragged=True, field=0.6, edge=0.5)])


@pytest.mark.parametrize("qpel", [0, 1])
def test_interlaced_svop(gpu, qpel):
    rng = np.random.default_rng(700 + qpel)
    check(gpu, [I.ilace_picture(rng, 23, 14, qpel=qpel, sprite=True, field=0.4)])


def test_stacked_1080_422(gpu):
    """sixteen 1920x1088 4:2:2 pictures in one call: frame P and B, first and second top / bottom fields"""
    pics = []
    for i in range(16):
        rng = np.random.default_rng(800 + i)
        structure = (M.FRAME, M.TOP, M.BOTTOM, M.FRAME)[i & 3]
        pics.append(I.cf_picture(rng, 2, 120, 68, structure=structure, first_field=(i >> 2) & 1, b=(i >> 3) & 1, no_rnd=i & 1,
                                 far=0.02, edge=0.05))
    check(gpu, pics)


def test_all_kinds_in_one_call(gpu):
    """4:2:0, 4:2:2, 4:4:4, interlaced MPEG-4 and an interlaced S-VOP in one call"""
    rng = np.random.default_rng(900)
    pics = [I.cf_picture(rng, cf, 11, 7, b=1) for cf in (1, 2, 3)]
    pics += [I.ilace_picture(rng, 11, 7, qpel=1, b=1), I.ilace_picture(rng, 11, 7, sprite=True)]
    check(gpu, pics)


# ------------------------------------------------------------------------------------------------------------------------------- flushes

def flush(gpu, checker, pics, xvid):
    """ff_mpv_flush_pictures_cuda over the pictures and a decoder's residual for them, against the chained checker; the coefficient
    arenas (every batch runs with clear) are compared too"""
    from libav_b200 import device
    batches = I.residual(checker, pics, np.random.default_rng(17), xvid=xvid)
    want = [I.run_ref(p) for p in pics]
    keeps = M.apply_residual(checker, M.xvid_checker(), want, batches)
    g = I.GpuPics(pics)
    res = M.GpuResidual(g, batches)
    w = res.work(g)
    gpu.check(gpu.lib.ff_mpv_flush_pictures_cuda(C.byref(w), None), "ff_mpv_flush_pictures_cuda")
    device.sync()
    got = g.download()
    for i in range(len(pics)):
        d = M.first_diff(got[i], want[i])
        assert d is None, (i, d)
    for b, d_b, keep in zip(batches, res.blocks, keeps):
        after = d_b.download(np.int16, b["blocks"].shape)
        assert not after[keep].any() and np.array_equal(after[~keep], b["blocks"][~keep])
    assert g.rejected() == 0


def test_flush_422_1080i(gpu, checker):
    """4:2:2 1080i: frame pictures with field-DCT luma and chroma batches, and field pictures"""
    pics = [I.cf_picture(np.random.default_rng(1000 + i), 2, 120, 68, structure=(M.FRAME, M.TOP)[i & 1], b=i >> 1, far=0.02, edge=0.05)
            for i in range(4)]
    flush(gpu, checker, pics, xvid=False)


def test_flush_444(gpu, checker):
    """4:4:4 frame and field pictures: twelve blocks per macroblock"""
    pics = [I.cf_picture(np.random.default_rng(1100 + i), 3, 23, 14, structure=(M.FRAME, M.BOTTOM)[i], b=i) for i in range(2)]
    flush(gpu, checker, pics, xvid=False)


def test_flush_interlaced_mpeg4_xvid(gpu, checker):
    """interlaced MPEG-4 with the Xvid IDCT (intra blocks through the fused h263_intra dequantiser) and field DCT"""
    pics = [I.ilace_picture(np.random.default_rng(1200 + i), 45, 36, qpel=i & 1, b=i >> 1, field=0.5) for i in range(4)]
    flush(gpu, checker, pics, xvid=True)
