"""The 8-bit H.264 batch calls against the reference on the edge cases of tests/h264_edge_cases.py, under every kernel the launchers can
pick: the defaults, and the fallbacks forced by their knobs (mc_variant = 2, residual_variant = 2) and reached by the inputs that need
them.  Pictures sit in decoder layout inside poisoned allocations: besides the pixels and the consumed coefficient arena, every byte
outside the picture rectangles must come back unchanged.

The inputs that send a call to its fallback kernel (libav_b200/csrc):
  MC        h264_mc.cu:118 luma plane or linesize not 4-byte aligned (pad2, shift1, shift2), :119 chroma plane or uvlinesize odd
            (odd_uv, odd_cb), :120 odd pic_w / pic_h; inside the default kernel, a reference plane off 4-byte alignment sends every
            block down the EDGE path (:73, ref1)
  residual  h264_residual.cu:171 coeff_stride % 8 (772) or an arena off 16-byte alignment (+2 bytes), :172 planes or line sizes off
            4-byte alignment (pad2, shift1, shift2, odd_uv); coeff_stride 776 keeps the default kernel at a stride other than 768
  deblock   h264dsp.cu:274 refuses planes and line sizes off 4-byte alignment"""
import contextlib
import ctypes as C

import numpy as np
import pytest

from libav_b200 import synth, tables
import h264_edge_cases as ec
import h264_util as hu

pytestmark = pytest.mark.gpu
MB_W, MB_H = 12, 8
TIGHT = ec.Layout("tight", 0, 0)
MC_KNOBS = [{}, {"mc_variant": 2}]
RES_KNOBS = [{}, {"residual_variant": 2}]
knob_id = lambda k: ",".join("%s=%d" % kv for kv in k.items()) or "default"


def _dev(a):
    from libav_b200 import device
    return device.DevBuf.from_numpy(np.ascontiguousarray(a))


@contextlib.contextmanager
def tuned(gpu, knobs):
    try:
        for k, v in knobs.items():
            gpu.lib.avb200_set_tuning(k.encode(), v)
        yield
    finally:
        for k in knobs:
            gpu.lib.avb200_set_tuning(k.encode(), 0)


class Placed:
    """planes placed by a Layout, uploaded whole (poison included); ptrs = the pictures' first samples on the device"""

    def __init__(self, lay, planes, ref=False):
        self.host = [lay.place(p, chroma=i > 0, ref=ref) for i, p in enumerate(planes)]
        self.dev = [_dev(b) for b, _ in self.host]
        self.ptrs = [d.ptr + ec.Layout.origin(b, v) for d, (b, v) in zip(self.dev, self.host)]
        self.ls = [v.strides[0] for _, v in self.host]

    def check(self, want, what=""):
        for (b, v), d, w, name in zip(self.host, self.dev, want, ("y", "cb", "cr")):
            b[...] = d.download(np.uint8, b.shape)
            ec.Layout.check(b, v, w, (what, name))


# ---- motion compensation ----
@pytest.fixture(scope="module")
def mc_case(checker):
    refs = [synth.h264_picture(MB_W, MB_H, seed=81), synth.h264_picture(MB_W, MB_H, seed=82)]
    dst = synth.h264_picture(MB_W, MB_H, seed=83)
    rec = ec.mc_records(MB_W, MB_H, seed=84)
    return refs, dst, rec, ec.oracle_mc(checker, rec, refs, dst)


def run_mc(gpu, rec, refs, dst, lay, pw, ph, knobs):
    from libav_b200 import device
    d, r = Placed(lay, dst), [Placed(lay, p, ref=True) for p in refs]
    planes, d_rec = _dev(np.array([p.ptrs for p in r], np.uint64)), _dev(rec)
    with tuned(gpu, knobs):
        gpu.check(gpu.lib.ff_h264_mc_batch_cuda(d_rec.ptr, rec.shape[0], planes.ptr, *d.ptrs, d.ls[0], d.ls[1], pw, ph, None))
        device.sync()
    for p, want in zip(r, refs):
        p.check(want, "reference")
    return d


@pytest.mark.parametrize("lay", [TIGHT, ec.PAD4, ec.PAD2, ec.SHIFT1, ec.SHIFT2, ec.ODD_UV, ec.ODD_CB, ec.REF1], ids=repr)
@pytest.mark.parametrize("knobs", MC_KNOBS, ids=knob_id)
def test_mc_far_vectors_in_decoder_layout(gpu, mc_case, lay, knobs):
    refs, dst, rec, want = mc_case
    run_mc(gpu, rec, refs, dst, lay, 16 * MB_W, 16 * MB_H, knobs).check(want)


@pytest.mark.parametrize("pw,ph", [(16 * MB_W - 1, 16 * MB_H), (16 * MB_W, 16 * MB_H - 1), (16 * MB_W - 3, 16 * MB_H - 3)])
def test_mc_odd_picture_size(gpu, checker, mc_case, pw, ph):
    refs, dst, rec, _ = mc_case
    run_mc(gpu, rec, refs, dst, ec.PAD4, pw, ph, {}).check(ec.oracle_mc(checker, rec, refs, dst, pw, ph))


@pytest.mark.parametrize("knobs", MC_KNOBS, ids=knob_id)
def test_mc_any_record_order_and_batch_size(gpu, checker, mc_case, knobs):
    refs, dst, rec, want = mc_case
    perm = rec[np.random.default_rng(6).permutation(rec.shape[0])]
    run_mc(gpu, perm, refs, dst, ec.PAD4, 16 * MB_W, 16 * MB_H, knobs).check(want, "permuted")
    for n in (1, 31, 33, 129):
        sub = rec[np.sort(np.random.default_rng(n).choice(rec.shape[0], n, replace=False))]
        run_mc(gpu, sub, refs, dst, ec.PAD4, 16 * MB_W, 16 * MB_H, knobs).check(ec.oracle_mc(checker, sub, refs, dst), n)


@pytest.mark.parametrize("knobs", MC_KNOBS, ids=knob_id)
def test_mc_stacked_pictures_far_vectors(gpu, checker, knobs):
    """two pictures stacked in one call, vectors up to the level limits in both directions: clamping stops at each picture's seam"""
    mb_w, mb_h, P = 6, 4, 2
    H = 16 * mb_h
    refs = [[synth.h264_picture(mb_w, mb_h, seed=90 + 2 * k + j) for j in range(2)] for k in range(P)]
    dsts = [synth.h264_picture(mb_w, mb_h, seed=95 + k) for k in range(P)]
    recs, wants = [], []
    for k in range(P):
        rec = ec.mc_records(mb_w, mb_h, seed=97 + k, band=0)
        wants.append(ec.oracle_mc(checker, rec, refs[k], dsts[k]))
        rec = rec.copy(); rec["y"] += k * H; recs.append(rec)
    cat = lambda planes: [np.concatenate([p[i] for p in planes]) for i in range(3)]
    stacked_refs = [cat([refs[k][j] for k in range(P)]) for j in range(2)]
    run_mc(gpu, np.concatenate(recs), stacked_refs, cat(dsts), ec.PAD4, 16 * mb_w, H, knobs).check(cat(wants))


# ---- residual ----
@pytest.fixture(scope="module")
def res_case(checker):
    mb_w, mb_h = 9, 6
    rec, coeffs, nnzc = ec.residual_records(mb_w, mb_h, seed=61)
    pic = synth.h264_picture(mb_w, mb_h, seed=62)
    want, want_co = [p.copy() for p in pic], coeffs.copy()
    hu.oracle_residual(checker, rec, want_co, nnzc, *want)
    return mb_w, rec, coeffs, nnzc, pic, want, want_co


@pytest.mark.parametrize("lay,shift,stride", [(TIGHT, 0, 768), (ec.PAD4, 0, 768), (ec.PAD2, 0, 768), (ec.SHIFT1, 0, 768),
                                              (ec.SHIFT2, 0, 768), (ec.ODD_UV, 0, 768), (ec.PAD4, 2, 768), (ec.PAD4, 0, 772),
                                              (ec.PAD4, 0, 776)], ids=lambda v: repr(v))
@pytest.mark.parametrize("knobs", RES_KNOBS, ids=knob_id)
def test_residual_wraparound_and_dispatch(gpu, res_case, lay, shift, stride, knobs):
    from libav_b200 import device
    mb_w, rec, coeffs, nnzc, pic, want, want_co = res_case
    n = coeffs.shape[0]
    d = Placed(lay, pic)
    r2 = ec.relayout_residual(rec, 16 * mb_w, d.ls[0], d.ls[1])
    arena = np.full(shift + 2 * n * stride + 16, 0x5A, np.uint8)               # the arena `shift` bytes into its allocation
    arena[shift:shift + 2 * n * stride].view(np.int16).reshape(n, stride)[:, :768] = coeffs
    d_rec, d_nz, d_co = _dev(r2), _dev(nnzc), _dev(arena)
    with tuned(gpu, knobs):
        gpu.check(gpu.lib.ff_h264_idct_add_mb_batch_cuda(d_rec.ptr, n, d_co.ptr + shift, stride, d_nz.ptr, *d.ptrs, d.ls[0], d.ls[1], None))
        device.sync()
    d.check(want)
    got = d_co.download(np.uint8, arena.shape)
    co = got[shift:shift + 2 * n * stride].copy().view(np.int16).reshape(n, stride)
    assert np.array_equal(co[:, :768], want_co), np.argwhere(co[:, :768] != want_co)[:5].tolist()
    assert (co[:, 768:] == 0x5A5A).all() and (got[:shift] == 0x5A).all() and (got[shift + 2 * n * stride:] == 0x5A).all()


# ---- weighted prediction ----
@pytest.mark.parametrize("lay", [TIGHT, ec.PAD2, ec.SHIFT1], ids=repr)
@pytest.mark.parametrize("bi", [0, 1])
def test_weight_every_corner(gpu, checker, lay, bi):
    from libav_b200 import device
    rec, plane, src = ec.weight_records(bi, seed=43)
    want = plane.copy()
    hu.oracle_weight(checker, rec, want, src if bi else None)
    assert (want == 0).any() and (want == 255).any()
    lp, ls_ = lay.place(plane), lay.place(src)
    d_pl, d_src = _dev(lp[0]), _dev(ls_[0])
    ls = lp[1].strides[0]
    r2 = rec.copy(); r2["off"] = ec.relayout_offsets(rec["off"], plane.shape[1], ls)
    d_rec = _dev(r2)
    gpu.check(gpu.lib.ff_h264_weight_batch_cuda(d_rec.ptr, rec.shape[0], d_pl.ptr + ec.Layout.origin(*lp),
                                                d_src.ptr + ec.Layout.origin(*ls_) if bi else None, ls, None))
    device.sync()
    lp[0][...] = d_pl.download(np.uint8, lp[0].shape)
    ec.Layout.check(*lp, want)
    ls_[0][...] = d_src.download(np.uint8, ls_[0].shape)
    ec.Layout.check(*ls_, src, "second prediction")


# ---- deblocking ----
def deblock_case(checker, mb_w, mb_h, seed):
    rec = ec.deblock_records(mb_w, mb_h, seed=seed)
    pic = [ec.blocky((16 * mb_h, 16 * mb_w), seed + 1), ec.blocky((8 * mb_h, 8 * mb_w), seed + 2), ec.blocky((8 * mb_h, 8 * mb_w), seed + 3)]
    want = [p.copy() for p in pic]
    hu.oracle_deblock(checker, rec, mb_w, mb_h, *want)
    assert (np.abs(want[0].astype(int) - pic[0]) > 12).sum() > 50              # the large-tc and strong filters did act
    return rec, pic, want


@pytest.mark.parametrize("lay", [TIGHT, ec.PAD4], ids=repr)
def test_deblock_high_qp_in_decoder_layout(gpu, checker, lay):
    from libav_b200 import device
    mb_w, mb_h = 9, 6
    rec, pic, want = deblock_case(checker, mb_w, mb_h, 55)
    d, d_rec, prog = Placed(lay, pic), _dev(rec), device.DevBuf(8 * mb_h)
    gpu.check(gpu.lib.ff_h264_deblock_picture_cuda(d_rec.ptr, mb_w, mb_h, *d.ptrs, d.ls[0], d.ls[1], prog.ptr, None))
    device.sync()
    d.check(want)


def test_deblock_batch_high_qp_in_decoder_layout(gpu, checker):
    from libav_b200 import device
    mb_w, mb_h, P = 7, 4, 2
    cases = [deblock_case(checker, mb_w, mb_h, 65 + 10 * k) for k in range(P)]
    cat = lambda i, j: np.concatenate([c[i][j] for c in cases])
    d = Placed(ec.PAD4, [cat(1, j) for j in range(3)])
    d_rec, prog = _dev(np.concatenate([c[0] for c in cases])), device.DevBuf(8 * mb_h * P)
    gpu.check(gpu.lib.ff_h264_deblock_batch_cuda(d_rec.ptr, mb_w, mb_h, P, *d.ptrs, d.ls[0], d.ls[1], prog.ptr, None))
    device.sync()
    d.check([cat(2, j) for j in range(3)])


@pytest.mark.parametrize("lay", [ec.PAD2, ec.SHIFT1, ec.ODD_UV], ids=repr)
def test_deblock_refuses_unaligned_planes(gpu, lay):
    from libav_b200 import device
    mb_w, mb_h = 4, 3
    pic = synth.h264_picture(mb_w, mb_h, seed=3)
    d, d_rec, prog = Placed(lay, pic), _dev(np.zeros(mb_w * mb_h, synth.DEBLOCK_DT)), device.DevBuf(8 * mb_h)
    for call in (lambda: gpu.lib.ff_h264_deblock_picture_cuda(d_rec.ptr, mb_w, mb_h, *d.ptrs, d.ls[0], d.ls[1], prog.ptr, None),
                 lambda: gpu.lib.ff_h264_deblock_batch_cuda(d_rec.ptr, mb_w, mb_h, 1, *d.ptrs, d.ls[0], d.ls[1], prog.ptr, None)):
        assert call() == -1
        assert "4-byte aligned" in gpu.last_error()
        gpu.lib.avb200_clear_error()
    device.sync()
    d.check(pic)


# ---- the flush point in decoder layout ----
def flush_batch(works, pics, refs, mb_w, mb_h, lay=ec.PAD4, c422=0):
    """works (test_gpu_h264flush.picture_work) and their pictures stacked into one FFH264PictureWork, planes and reference planes placed
    by `lay`: returns (work, placed pictures, the device buffers work points to).  Offsets of the works are tight byte offsets, so
    16-bit pictures (uint16 planes, int32 coefficients) and 4:2:2 ones (c422: 16 chroma rows per macroblock) stack the same way; the
    caller sets work.bit_depth / chroma_format_idc.  A work with "deblock" = (records, 4:2:2 records or None) in place of "info" hands
    the loop filter its records directly."""
    from libav_b200 import device
    P = len(works)
    W, H = 16 * mb_w * pics[0][0].itemsize, 16 * mb_h
    CH = H if c422 else H // 2
    cat = lambda planes: [np.concatenate([p[i] for p in planes]) for i in range(3)]
    d = Placed(lay, cat(pics))
    r = [Placed(lay, [np.concatenate([p] * P) for p in rp], ref=True) for rp in refs]
    ls, uvls = d.ls[0], d.ls[1]
    mc, res, wrec = [], [], []
    for k, w in enumerate(works):
        m = w["mc"].copy(); m["y"] += H * k; mc.append(m)
        rr = ec.relayout_residual(w["res"], W, ls, uvls); rr["luma_off"] += H * k * ls; rr["chroma_off"] += CH * k * uvls; res.append(rr)
        t = w["weight"].copy(); t["off"] = ec.relayout_offsets(t["off"], W, ls) + H * k * ls; wrec.append(t)
    mc, res, wrec = np.concatenate(mc), np.concatenate(res), np.concatenate(wrec)
    n = mb_w * mb_h * P
    catw = lambda k: np.concatenate([w[k] for w in works])
    dv = dict(planes=_dev(np.array([p.ptrs for p in r], np.uint64)), mc=_dev(mc), res=_dev(res), w=_dev(wrec), co=_dev(catw("coeffs")),
              nz=_dev(catw("nnzc")), dc=_dev(catw("dc")), ldc=_dev(catw("luma_dc")), intra=_dev(catw("intra")), rec=device.DevBuf(n * 104),
              prog=device.DevBuf(4 * 2 * mb_h * P), refs=r)
    work = tables.FFH264PictureWork()
    if "info" in works[0]:
        infos = [w["info"] for w in works]
        catinfo = lambda k: np.concatenate([i[k] for i in infos], axis=0)
        keep = {k: _dev(catinfo(k)) for k in ("mb_type", "qscale", "nnz", "cbp", "slice_table", "mv0", "mv1", "ref0", "ref1")}
        keep["sp"] = _dev(infos[0]["slice_params"]); keep["cq"] = _dev(infos[0]["chroma_qp_table"])
        info = tables.FFH264DeblockInfo(mb_w, mb_h, P, keep["mb_type"].ptr, keep["qscale"].ptr, keep["nnz"].ptr, keep["cbp"].ptr, keep["slice_table"].ptr,
                                        (C.c_void_p * 2)(keep["mv0"].ptr, keep["mv1"].ptr), (C.c_void_p * 2)(keep["ref0"].ptr, keep["ref1"].ptr),
                                        keep["sp"].ptr, infos[0]["n_slices"], keep["cq"].ptr, infos[0]["cabac"], infos[0]["t8x8"])
        dv.update(keep=keep, info=info)
        work.deblock_info = C.pointer(info)
    else:
        dv["rec"] = _dev(np.concatenate([w["deblock"][0] for w in works]))
        if c422:
            dv["ext"] = _dev(np.concatenate([w["deblock"][1] for w in works]))
            work.deblock_chroma422 = dv["ext"].ptr
    work.mb_w, work.mb_h, work.n_pictures = mb_w, mb_h, P
    work.luma, work.cb, work.cr = d.ptrs
    work.linesize, work.uvlinesize = ls, uvls
    work.mc, work.n_mc, work.refs = dv["mc"].ptr, mc.shape[0], dv["planes"].ptr
    work.weight[0], work.n_weight[0] = dv["w"].ptr, wrec.shape[0]
    work.coeffs, work.coeff_stride, work.nnzc = dv["co"].ptr, 768, dv["nz"].ptr
    work.dc, work.luma_dc, work.residual, work.intra = dv["dc"].ptr, dv["ldc"].ptr, dv["res"].ptr, dv["intra"].ptr
    work.deblock_records, work.progress = dv["rec"].ptr, dv["prog"].ptr
    return work, d, dv


def test_flush_in_decoder_layout(gpu, checker):
    """ff_h264_flush_pictures_cuda over two stacked pictures whose planes have line sizes wider than the picture: every stage's
    records address the decoder's layout, the checker runs on tight copies"""
    from libav_b200 import device
    from test_gpu_h264flush import picture_work, oracle_chain
    mb_w, mb_h, P = 20, 12, 2
    refs = [synth.h264_picture(mb_w, mb_h, seed=11), synth.h264_picture(mb_w, mb_h, seed=12)]
    works = [picture_work(mb_w, mb_h, 300 + 100 * k, 0.25) for k in range(P)]
    pics = [synth.h264_picture(mb_w, mb_h, seed=70 + k) for k in range(P)]
    want, want_co = [], []
    for w, p in zip(works, pics):
        wp = [x.copy() for x in p]
        want_co.append(oracle_chain(checker, w, refs, mb_w, mb_h, *wp))
        want.append(wp)
    work, d, dv = flush_batch(works, pics, refs, mb_w, mb_h)
    gpu.check(gpu.lib.ff_h264_flush_pictures_cuda(C.byref(work), None))
    device.sync()
    d.check([np.concatenate([w[i] for w in want]) for i in range(3)])
    assert np.array_equal(dv["co"].download(np.int16, (mb_w * mb_h * P, 768)), np.concatenate(want_co))
