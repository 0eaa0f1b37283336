"""The 9 / 10-bit and 4:2:2 H.264 batch calls of h264_hbd_batch.cu against the reference on the edge cases of tests/h264_edge_cases.py,
on the GPU: far, limit and outside vectors under both MC kernels (mc_hbd_staged 0: patches staged in shared memory; 2: clamped global
loads), pictures stacked in one call so that clamping has to stop at every seam, shuffled put / avg records; coefficients at both ends
of the legal range and every dispatch rule, including the lower 4:2:2 chroma blocks; every weight corner; DC transforms at the largest
qmul; the deblocking wavefront with high-qp records on blocky content from one macroblock to two stacked 1920x1088 pictures; the flush
point on stacked pictures in decoder layout; and the misaligned arguments the 16-bit calls refuse.  Pictures sit in decoder layout
inside poisoned allocations: besides the pixels and the consumed coefficient arena, every byte outside the pictures must come back
unchanged.  The CPU runs the same cases through the host-compiled kernels (tests/test_h264_hbd_edges_cpu.py)."""
import functools

import numpy as np
import pytest

from libav_b200 import synth
import h264_edge_cases as ec
import h264_hbd_util as hh
from test_gpu_h264_edges import Placed, tuned, flush_batch
from test_h264_hbd_edges_cpu import (CASES, MB_W, MB_H, MC_LAYOUTS, REFUSED, case_id, mc_case, oracle_mc, stacked_mc_case, residual_case,
                                     run_residual, weight_case, run_weight, dc_case, run_dc)

pytestmark = pytest.mark.gpu
TIGHT = ec.Layout("tight", 0, 0)
STAGED = [0, 2]


def _dev(a):
    from libav_b200 import device
    return device.DevBuf.from_numpy(np.ascontiguousarray(a))


def on_device(placed):
    """(device buffers, pointers at the pictures' first samples) for (allocation, view) pairs"""
    devs = [_dev(b) for b, _ in placed]
    return devs, [dv.ptr + ec.Layout.origin(b, v) for dv, (b, v) in zip(devs, placed)]


def back(devs, placed):
    from libav_b200 import device
    device.sync()
    for dv, (b, _) in zip(devs, placed):
        b[...] = dv.download(np.uint8, b.shape)


# ---- motion compensation ----
def run_mc(gpu, bits, c422, rec, refs, dst, lay, pw, ph, staged):
    from libav_b200 import device
    d, r = Placed(lay, dst), [Placed(lay, p, ref=True) for p in refs]
    planes, d_rec = _dev(np.array([p.ptrs for p in r], np.uint64)), _dev(rec)
    with tuned(gpu, {"mc_hbd_staged": staged}):
        gpu.check(gpu.lib.ff_h264_mc_batch_hbd_cuda(bits, 1 + c422, d_rec.ptr, rec.shape[0], planes.ptr, *d.ptrs, d.ls[0], d.ls[1], pw, ph, None))
        device.sync()
    for p, want in zip(r, refs):
        p.check(want, "reference")
    return d


@pytest.fixture(scope="module", params=CASES, ids=case_id)
def mc_far(request, checker):
    bits, c422 = request.param
    return (bits, c422) + mc_case(checker, bits, c422, seed=140 + bits + 5 * c422)


@pytest.mark.parametrize("staged", STAGED)
@pytest.mark.parametrize("lay", MC_LAYOUTS, ids=repr)
def test_mc_far_vectors_in_decoder_layout(gpu, mc_far, lay, staged):
    bits, c422, refs, dst, rec, want = mc_far
    run_mc(gpu, bits, c422, rec, refs, dst, lay, 16 * MB_W, 16 * MB_H, staged).check(want)


@pytest.mark.parametrize("staged", STAGED)
def test_mc_any_record_order_and_batch_size(gpu, checker, mc_far, staged):
    bits, c422, refs, dst, rec, want = mc_far
    perm = rec[np.random.default_rng(6).permutation(rec.shape[0])]
    run_mc(gpu, bits, c422, perm, refs, dst, ec.PAD2, 16 * MB_W, 16 * MB_H, staged).check(want, "permuted")
    for n in (1, 7, 33, 130):
        sub = perm[:n]
        run_mc(gpu, bits, c422, sub, refs, dst, ec.PAD2, 16 * MB_W, 16 * MB_H, staged).check(oracle_mc(checker, bits, c422, sub, refs, dst), n)


@pytest.mark.parametrize("staged", STAGED)
@pytest.mark.parametrize("P", [2, 3])
@pytest.mark.parametrize("case", CASES, ids=case_id)
def test_mc_stacked_pictures_far_vectors(gpu, checker, case, P, staged):
    bits, c422 = case
    rec, refs, dst, want, mb_w, H = stacked_mc_case(checker, bits, c422, P)
    run_mc(gpu, bits, c422, rec, refs, dst, ec.PAD4, 16 * mb_w, H, staged).check(want)


# ---- residual, weighted prediction, DC transforms ----
@pytest.fixture(scope="module", params=CASES, ids=case_id)
def res_case(request, checker):
    bits, c422 = request.param
    return bits, c422, residual_case(checker, bits, c422, seed=161 + bits + 3 * c422)


@pytest.mark.parametrize("lay,stride", [(TIGHT, 768), (ec.PAD4, 776), (ec.PAD2, 768), (ec.SHIFT2, 768), (ec.CSHIFT2, 770)],
                         ids=lambda v: repr(v))
def test_residual_range_ends_and_dispatch(gpu, res_case, lay, stride):
    bits, c422, case = res_case

    def call(bits, idc, rec, arena, stride, nnzc, d):
        devs, ptrs = on_device(d)
        d_rec, d_co, d_nz = _dev(rec), _dev(arena), _dev(nnzc)
        gpu.check(gpu.lib.ff_h264_idct_add_mb_batch_hbd_cuda(bits, idc, d_rec.ptr, rec.shape[0], d_co.ptr, stride, d_nz.ptr, *ptrs,
                                                             d[0][1].strides[0], d[1][1].strides[0], None))
        back(devs, d)
        arena[...] = d_co.download(arena.dtype, arena.shape)
        return 0
    run_residual(call, bits, c422, case, lay, stride)


@pytest.mark.parametrize("lay", [TIGHT, ec.PAD2, ec.SHIFT2], ids=repr)
@pytest.mark.parametrize("bi", [0, 1])
@pytest.mark.parametrize("bits", [9, 10])
def test_weight_every_corner(gpu, checker, bits, bi, lay):
    def call(bits, rec, lp, ls_, ls):
        placed = [lp] + ([ls_] if ls_ else [])
        devs, ptrs = on_device(placed)
        d_rec = _dev(rec)
        gpu.check(gpu.lib.ff_h264_weight_batch_hbd_cuda(bits, d_rec.ptr, rec.shape[0], ptrs[0], ptrs[1] if ls_ else None, ls, None))
        back(devs, placed)
        return 0
    run_weight(call, bits, bi, weight_case(checker, bits, bi, seed=143 + bi), lay)


@pytest.mark.parametrize("c422", [0, 1])
@pytest.mark.parametrize("bits", [9, 10])
def test_dc_range_ends_and_largest_qmul(gpu, checker, bits, c422):
    from libav_b200 import device

    def call(idc, rec, arena, stride, luma_dc):
        d_rec, d_co, d_dc = _dev(rec), _dev(arena), _dev(luma_dc)
        gpu.check(gpu.lib.ff_h264_dc_dequant_batch_hbd_cuda(idc, d_rec.ptr, rec.shape[0], d_co.ptr, stride, d_dc.ptr, None))
        device.sync()
        arena[...] = d_co.download(np.int32, arena.shape)
        return 0
    run_dc(call, c422, dc_case(checker, bits, c422, seed=107 + bits + c422))


# ---- deblocking ----
DEBLOCK_CASES = [(9, 0), (10, 0), (8, 1), (9, 1), (10, 1)]
SHAPES = [(1, 1, 1), (1, 37, 1), (45, 1, 1), (120, 68, 2)]          # (mb_w, mb_h, pictures): 120 x 68 = 1920 x 1088, 68 rows > 16 warps


@functools.lru_cache(maxsize=None)
def deblock_work(mb_w, mb_h, k):
    return ec.deblock422_records(mb_w, mb_h, seed=300 + 7 * mb_w + mb_h + 100 * k)


@pytest.mark.parametrize("shape", SHAPES, ids=lambda s: "%dx%dx%d" % s)
@pytest.mark.parametrize("case", DEBLOCK_CASES, ids=case_id)
def test_deblock_high_qp_blocky_in_decoder_layout(gpu, checker, case, shape):
    """ff_h264_deblock_batch_hbd_cuda (4:2:0) / ff_h264_deblock_batch_422_cuda: records over the whole qp range with slice offsets on
    content whose steps reach 2^bits - 1, pictures stacked, planes at +2 bytes with padded pitches; every picture must equal its
    own serial result"""
    from libav_b200 import device
    bits, c422 = case
    mb_w, mb_h, P = shape
    top, ch = (1 << bits) - 1, 16 * mb_h if c422 else 8 * mb_h
    pics, wants, recs, exts = [], [], [], []
    for k in range(P):
        rec, ext, qps = deblock_work(mb_w, mb_h, k)
        pic = [ec.blocky((16 * mb_h, 16 * mb_w), 20 + 3 * k, bits), ec.blocky((ch, 8 * mb_w), 21 + 3 * k, bits), ec.blocky((ch, 8 * mb_w), 22 + 3 * k, bits)]
        want = [p.copy() for p in pic]
        if c422:
            hh.oracle_deblock422(checker, bits, rec, ext, mb_w, mb_h, *want)
        else:
            hh.oracle_deblock(checker, bits, rec, mb_w, mb_h, *want)
        if mb_w * mb_h >= 32:                                          # (one macroblock has too few edges to promise anything)
            assert ec.high_qp_edges_changed(qps, mb_w, mb_h, pic[0], want[0]) > 16 * mb_w * mb_h // 4
        if mb_w * mb_h >= 1000:                                       # steps from 0 to 2^bits - 1 under the wavefront
            assert (pic[0] == 0).any() and (pic[0] == top).any()
        pics.append(pic); wants.append(want); recs.append(rec); exts.append(ext)
    cat = lambda planes: [np.concatenate([p[i] for p in planes]) for i in range(3)]
    d, d_rec = Placed(ec.SHIFT2, cat(pics)), _dev(np.concatenate(recs))
    if c422:
        d_ext = _dev(np.concatenate(exts))
        gpu.check(gpu.lib.ff_h264_deblock_batch_422_cuda(bits, d_rec.ptr, d_ext.ptr, mb_w, mb_h, P, *d.ptrs, d.ls[0], d.ls[1], None))
    else:
        gpu.check(gpu.lib.ff_h264_deblock_batch_hbd_cuda(bits, d_rec.ptr, mb_w, mb_h, P, *d.ptrs, d.ls[0], d.ls[1], None))
    device.sync()
    d.check(cat(wants))


# ---- the flush point in decoder layout ----
def flush_work(checker, mb_w, mb_h, bits, c422, k, refs):
    """one picture's records for every stage at 9 / 10 bit from the edge generators (intra macroblocks from hh.intra_work), the picture
    and the chained checker's result: (work, picture, wanted picture, wanted arena)"""
    rng = np.random.default_rng(500 + k)
    n = mb_w * mb_h
    top = (1 << bits) - 1
    ch = 16 * mb_h if c422 else 8 * mb_h
    pic = [ec.blocky((16 * mb_h, 16 * mb_w), 60 + 3 * k, bits), ec.blocky((ch, 8 * mb_w), 61 + 3 * k, bits), ec.blocky((ch, 8 * mb_w), 62 + 3 * k, bits)]
    irec, ico, inz = hh.intra_work(mb_w, mb_h, bits, seed=70 + k, p_intra=0.25, c422=c422)
    res, co, nz = ec.residual_records(mb_w, mb_h, seed=80 + k, bits=bits, c422=c422)
    intra = irec["kind"] != 0
    res["luma_mode"][intra] = 3; res["chroma"][intra] = 0
    co[intra] = ico[intra]; nz[intra] = inz[intra]
    mc = ec.mc_records(mb_w, mb_h, seed=90 + k, band=0)
    mc = mc[~intra[(mc["y"] // 16) * mb_w + mc["x"] // 16]]
    dc = np.zeros(n, ec.DC_DT)                 # luma_qmul < 900 and chroma_qmul <= 200 keep the reference's int arithmetic in range here
    dc["luma_qmul"] = np.where(~intra & (rng.random(n) < 0.3), rng.integers(16, 900, n), 0)
    dc["chroma_qmul"] = np.where(~intra[:, None] & (rng.random((n, 2)) < 0.5), rng.integers(16, 200, (n, 2)), 0)
    luma_dc = rng.integers(-(1 << (7 + bits)), 1 << (7 + bits), (n, 16)).astype(np.int32)
    wm = np.flatnonzero(~intra & (rng.random(n) < 0.4))
    wrec = np.zeros(wm.shape[0], synth.WEIGHT_DT)
    wrec["off"] = ((wm // mb_w) * 16 * 16 * mb_w + (wm % mb_w) * 16) * 2
    wrec["w"] = wrec["h"] = 16
    wrec["log2_denom"] = rng.integers(0, 8, wm.shape[0]); wrec["weight"] = rng.choice(ec.WEIGHTS, wm.shape[0]); wrec["offset"] = rng.choice(ec.OFFSETS, wm.shape[0])
    rec, ext, _ = ec.deblock422_records(mb_w, mb_h, seed=95 + k)
    want, want_co = [p.copy() for p in pic], co.copy()
    hh.oracle_mc(checker, bits, c422, mc, refs, *want)
    hh.oracle_weight(checker, bits, wrec, want[0])
    hh.oracle_dc(checker, bits, c422, dc, want_co, luma_dc)
    hh.oracle_residual(checker, bits, c422, res, want_co, nz, *want)
    hh.oracle_intra(checker, bits, irec, want_co, nz, mb_w, mb_h, *want, c422=c422)
    pre = want[0].copy()
    if c422:
        hh.oracle_deblock422(checker, bits, rec, ext, mb_w, mb_h, *want)
    else:
        hh.oracle_deblock(checker, bits, rec, mb_w, mb_h, *want)
    assert not np.array_equal(pre, want[0]) and (want[0] == 0).any() and (want[0] == top).any()
    work = dict(mc=mc, res=res, weight=wrec, coeffs=co, nnzc=nz, dc=dc, luma_dc=luma_dc, intra=irec, deblock=(rec, ext if c422 else None))
    return work, pic, want, want_co


@pytest.mark.parametrize("c422", [0, 1])
def test_flush_hbd_in_decoder_layout(gpu, checker, c422):
    """ff_h264_flush_pictures_cuda with bit_depth 10 over two stacked pictures whose planes have padded pitches: MC with far vectors ->
    weighted prediction -> DC transforms -> residual at the range ends -> intra -> high-qp loop filter, against the checker chained in
    the same order on tight copies"""
    import ctypes as C
    from libav_b200 import device
    bits, mb_w, mb_h, P = 10, 12, 8, 2
    refs = [hh.picture(mb_w, mb_h, bits, c422, seed=11 + j) for j in range(2)]
    cases = [flush_work(checker, mb_w, mb_h, bits, c422, k, refs) for k in range(P)]
    work, d, dv = flush_batch([c[0] for c in cases], [c[1] for c in cases], refs, mb_w, mb_h, ec.PAD2, c422)
    work.bit_depth, work.chroma_format_idc = bits, 1 + c422
    gpu.check(gpu.lib.ff_h264_flush_pictures_cuda(C.byref(work), None))
    device.sync()
    d.check([np.concatenate([c[2][i] for c in cases]) for i in range(3)])
    got = dv["co"].download(np.int32, (mb_w * mb_h * P, 768))
    assert np.array_equal(got, np.concatenate([c[3] for c in cases]))


# ---- refusals ----
@pytest.mark.parametrize("lay", REFUSED, ids=repr)
def test_refuses_odd_planes_and_pitches(gpu, lay):
    """16-bit samples at an odd address or with an odd pitch: every call returns -1, sets the error message and writes nothing"""
    from libav_b200 import device
    lib = gpu.lib
    pics = {c422: hh.picture(2, 2, 10, c422, seed=3) for c422 in (0, 1)}
    placed = {c422: Placed(lay, pics[c422]) for c422 in (0, 1)}
    rec = _dev(ec.mc_records(12, 8, seed=1)[:8])
    res, co, nz = _dev(np.zeros(4, synth.RESIDUAL_DT)), _dev(np.ones((4, 768), np.int32)), _dev(np.full((4, 120), 3, np.uint8))
    wrec = np.zeros(1, synth.WEIGHT_DT); wrec["w"] = wrec["h"] = 8; wrec["weight"] = 3
    d_w, dbk, d_ext = _dev(wrec), _dev(np.zeros(4, synth.DEBLOCK_DT)), _dev(np.zeros(4, ec.CHROMA422_DT))
    calls = []
    for c422, d in placed.items():
        planes = _dev(np.array([d.ptrs] * 2, np.uint64))
        odd = 0 if (d.ls[0] | d.ptrs[0]) & 1 else 1
        calls += [lambda d=d, c=c422, pl=planes: lib.ff_h264_mc_batch_hbd_cuda(10, 1 + c, rec.ptr, 8, pl.ptr, *d.ptrs, d.ls[0], d.ls[1], 32, 32, None),
                  lambda d=d, c=c422: lib.ff_h264_idct_add_mb_batch_hbd_cuda(10, 1 + c, res.ptr, 4, co.ptr, 768, nz.ptr, *d.ptrs, d.ls[0], d.ls[1], None),
                  lambda d=d, o=odd: lib.ff_h264_weight_batch_hbd_cuda(10, d_w.ptr, 1, d.ptrs[o], None, d.ls[o], None)]
        calls.append((lambda d=d: lib.ff_h264_deblock_batch_422_cuda(10, dbk.ptr, d_ext.ptr, 2, 2, 1, *d.ptrs, d.ls[0], d.ls[1], None)) if c422 else
                     (lambda d=d: lib.ff_h264_deblock_batch_hbd_cuda(10, dbk.ptr, 2, 2, 1, *d.ptrs, d.ls[0], d.ls[1], None)))
    for k, call in enumerate(calls):
        assert call() == -1, k
        assert "16-bit samples need even plane addresses and pitches" in gpu.last_error(), k
        lib.avb200_clear_error()
    device.sync()
    for c422, d in placed.items():
        d.check(pics[c422])
    assert (co.download(np.int32, (4, 768)) == 1).all()
