"""GPU parity for the batched H.264 calls on 9 / 10-bit and 4:2:2 pictures (libav_b200/csrc/h264_hbd_batch.cu) against the CPU oracle's
BIT_DEPTH > 8 instances applied macroblock by macroblock in the reference's order (tests/h264_hbd_util.py).  Sorted last: written after the
rest of the suite had been green on the GPU."""
import numpy as np
import pytest

from libav_b200 import synth
import h264_hbd_util as hh

pytestmark = pytest.mark.gpu
SIZES = [(3, 2), (7, 5), (20, 12)]


def _dev(a):
    from libav_b200 import device
    return device.DevBuf.from_numpy(a)


@pytest.mark.parametrize("bits,c422", [(9, 0), (9, 1), (10, 0), (10, 1), (8, 1)])
@pytest.mark.parametrize("mb_w,mb_h", SIZES)
def test_residual_batch_hbd(gpu, checker, mb_w, mb_h, bits, c422):
    from libav_b200 import device
    y, cb, cr = hh.picture(mb_w, mb_h, bits, c422, seed=5)
    rec, coeffs, nnzc = hh.residual_work(mb_w, mb_h, bits, c422, y, cb, seed=mb_w + bits)
    wy, wcb, wcr, wco = y.copy(), cb.copy(), cr.copy(), coeffs.copy()
    hh.oracle_residual(checker, bits, c422, rec, wco, nnzc, wy, wcb, wcr)
    assert not np.array_equal(wy, y) and not np.array_equal(wcb, cb)
    d = [_dev(x) for x in (rec, coeffs, nnzc, y, cb, cr)]
    gpu.check(gpu.lib.ff_h264_idct_add_mb_batch_hbd_cuda(bits, 1 + c422, d[0].ptr, rec.shape[0], d[1].ptr, 768, d[2].ptr, d[3].ptr, d[4].ptr, d[5].ptr,
                                                         y.strides[0], cb.strides[0], None))
    device.sync()
    assert np.array_equal(d[3].download(y.dtype, y.shape), wy)
    assert np.array_equal(d[4].download(y.dtype, cb.shape), wcb)
    assert np.array_equal(d[5].download(y.dtype, cr.shape), wcr)
    assert np.array_equal(d[1].download(coeffs.dtype, coeffs.shape), wco)      # consumed coefficients are zeroed identically


@pytest.mark.parametrize("staged", [0, 2])
@pytest.mark.parametrize("bits,c422", [(9, 0), (9, 1), (10, 0), (10, 1), (8, 1)])
@pytest.mark.parametrize("mb_w,mb_h", SIZES)
def test_mc_batch_hbd(gpu, checker, mb_w, mb_h, bits, c422, staged):
    """staged 0: the default kernel (patches staged in shared memory); 2: the clamped-global-load form of the same arithmetic (tests/hostsim/ runs it)"""
    from libav_b200 import device
    gpu.lib.avb200_set_tuning(b"mc_hbd_staged", staged)
    refs = [hh.picture(mb_w, mb_h, bits, c422, seed=11), hh.picture(mb_w, mb_h, bits, c422, seed=12)]
    rec = synth.h264_mc_work(mb_w, mb_h, seed=mb_h + bits, max_mv=64 if mb_w > 4 else 24, avg_second=True)
    y, cb, cr = hh.picture(mb_w, mb_h, bits, c422, seed=13)
    wy, wcb, wcr = y.copy(), cb.copy(), cr.copy()
    hh.oracle_mc(checker, bits, c422, rec, refs, wy, wcb, wcr)
    dref = [[_dev(p) for p in r] for r in refs]
    planes = np.array([[p.ptr for p in r] for r in dref], dtype=np.uint64)
    d_planes, d_rec = _dev(planes), _dev(rec)
    dy, dcb, dcr = _dev(y), _dev(cb), _dev(cr)
    gpu.check(gpu.lib.ff_h264_mc_batch_hbd_cuda(bits, 1 + c422, d_rec.ptr, rec.shape[0], d_planes.ptr, dy.ptr, dcb.ptr, dcr.ptr, y.strides[0], cb.strides[0],
                                                16 * mb_w, 16 * mb_h, None))
    device.sync()
    gpu.lib.avb200_set_tuning(b"mc_hbd_staged", 0)
    assert np.array_equal(dy.download(y.dtype, y.shape), wy)
    assert np.array_equal(dcb.download(y.dtype, cb.shape), wcb)
    assert np.array_equal(dcr.download(y.dtype, cr.shape), wcr)


@pytest.mark.parametrize("bits", [9, 10])
@pytest.mark.parametrize("mb_w,mb_h,slices,P", [(3, 2, 1, 1), (7, 5, 4, 2), (20, 12, 1, 3), (40, 36, 8, 2)])
def test_deblock_batch_hbd(gpu, checker, mb_w, mb_h, slices, P, bits):
    """P stacked pictures, rows of one picture as a wavefront inside one CTA: every picture must equal its own serial result"""
    from libav_b200 import device
    ys, cbs, crs, recs, want = [], [], [], [], []
    for k in range(P):
        y, cb, cr = hh.smooth_picture(mb_w, mb_h, bits, seed=100 * mb_w + k)
        rec = synth.h264_deblock_work(mb_w, mb_h, seed=slices + k, slices=slices)
        wy, wcb, wcr = y.copy(), cb.copy(), cr.copy()
        hh.oracle_deblock(checker, bits, rec, mb_w, mb_h, wy, wcb, wcr)
        assert not np.array_equal(wy, y) and not np.array_equal(wcb, cb)
        ys.append(y); cbs.append(cb); crs.append(cr); recs.append(rec); want.append((wy, wcb, wcr))
    Y, CB, CR, R = np.concatenate(ys), np.concatenate(cbs), np.concatenate(crs), np.concatenate(recs)
    d_rec, dy, dcb, dcr = _dev(R), _dev(Y), _dev(CB), _dev(CR)
    gpu.check(gpu.lib.ff_h264_deblock_batch_hbd_cuda(bits, d_rec.ptr, mb_w, mb_h, P, dy.ptr, dcb.ptr, dcr.ptr, Y.strides[0], CB.strides[0], None))
    device.sync()
    gy, gcb, gcr = dy.download(np.uint16, Y.shape), dcb.download(np.uint16, CB.shape), dcr.download(np.uint16, CR.shape)
    for k in range(P):
        assert np.array_equal(gy[16 * mb_h * k:16 * mb_h * (k + 1)], want[k][0]), k
        assert np.array_equal(gcb[8 * mb_h * k:8 * mb_h * (k + 1)], want[k][1]), k
        assert np.array_equal(gcr[8 * mb_h * k:8 * mb_h * (k + 1)], want[k][2]), k


def test_hbd_refusals(gpu):
    lib = gpu.lib
    assert lib.ff_h264_idct_add_mb_batch_hbd_cuda(8, 1, None, 0, None, 768, None, None, None, None, 64, 32, None) == -1
    assert lib.ff_h264_mc_batch_hbd_cuda(10, 3, None, 0, None, None, None, None, 64, 32, 16, 16, None) == -1
    assert lib.ff_h264_deblock_batch_hbd_cuda(10, None, 1, 1, 1, None, None, None, 64, 32, None) == -1
    lib.avb200_clear_error()


@pytest.mark.parametrize("bits", [8, 9, 10])
@pytest.mark.parametrize("mb_w,mb_h,slices,P", [(3, 2, 1, 1), (7, 5, 4, 2), (20, 12, 1, 3), (40, 36, 8, 2)])
def test_deblock_batch_422(gpu, checker, mb_w, mb_h, slices, P, bits):
    """chroma_format_idc 2: two 16-line vertical and four horizontal chroma edges per macroblock (8 / 9 / 10 bit), stacked pictures"""
    from libav_b200 import device
    dt = np.uint8 if bits == 8 else np.uint16
    ys, cbs, crs, recs, exts, want = [], [], [], [], [], []
    for k in range(P):
        y, cb, cr = hh.smooth_picture422(mb_w, mb_h, bits, seed=100 * mb_w + k)
        rec, ext = hh.deblock422_work(mb_w, mb_h, seed=slices + k, slices=slices)
        wy, wcb, wcr = y.copy(), cb.copy(), cr.copy()
        hh.oracle_deblock422(checker, bits, rec, ext, mb_w, mb_h, wy, wcb, wcr)
        assert not np.array_equal(wy, y) and not np.array_equal(wcb, cb)
        ys.append(y); cbs.append(cb); crs.append(cr); recs.append(rec); exts.append(ext); want.append((wy, wcb, wcr))
    Y, CB, CR, R, X = np.concatenate(ys), np.concatenate(cbs), np.concatenate(crs), np.concatenate(recs), np.concatenate(exts)
    d_rec, d_ext, dy, dcb, dcr = _dev(R), _dev(X), _dev(Y), _dev(CB), _dev(CR)
    gpu.check(gpu.lib.ff_h264_deblock_batch_422_cuda(bits, d_rec.ptr, d_ext.ptr, mb_w, mb_h, P, dy.ptr, dcb.ptr, dcr.ptr, Y.strides[0], CB.strides[0], None))
    device.sync()
    gy, gcb, gcr = dy.download(dt, Y.shape), dcb.download(dt, CB.shape), dcr.download(dt, CR.shape)
    for k in range(P):
        assert np.array_equal(gy[16 * mb_h * k:16 * mb_h * (k + 1)], want[k][0]), k
        assert np.array_equal(gcb[16 * mb_h * k:16 * mb_h * (k + 1)], want[k][1]), k
        assert np.array_equal(gcr[16 * mb_h * k:16 * mb_h * (k + 1)], want[k][2]), k


def test_chroma422_decisions(gpu, checker):
    """FFH264DeblockInfo.chroma422: the decisions of a 4:2:2 picture (h264_loopfilter.c:633,693-700) against the reference's own h264_loopfilter.c"""
    import ctypes as C
    from libav_b200 import device, tables
    from test_oracle_h264lf_cpu import C422_CASES, run422
    from test_gpu_h264lf import gpu_params
    for case in C422_CASES:
        for (mw, mh) in ((11, 9), (2, 5), (40, 17)):
            d = synth.h264_deblock_info(mw, mh, **case)
            want, want_ext = run422(checker, d)
            ext = device.DevBuf(52 * mw * mh); ext.fill(0xCD)
            got, _ = gpu_params(gpu, [d], chroma422=ext.ptr)
            bad = np.argwhere((got[:, :102] != want[:, :102]).any(axis=1))
            assert not len(bad), (case, mw, mh, bad[:4].ravel().tolist(), got[bad[0, 0]].tolist(), want[bad[0, 0]].tolist())
            gext = ext.download(np.uint8, (mw * mh, 52))
            bad = np.argwhere((gext[:, :50] != want_ext[:, :50]).any(axis=1))
            assert not len(bad), ("ext", case, mw, mh, bad[:4].ravel().tolist(), gext[bad[0, 0]].tolist(), want_ext[bad[0, 0]].tolist())


@pytest.mark.parametrize("bits", [9, 10])
def test_weight_and_dc_batch_hbd(gpu, checker, bits):
    from libav_b200 import device
    lib = gpu.lib

    def run_weight(b, rec, plane, src):
        d_rec, d_pl = _dev(rec), _dev(plane)
        d_src = _dev(src) if src is not None else None
        gpu.check(lib.ff_h264_weight_batch_hbd_cuda(b, d_rec.ptr, rec.shape[0], d_pl.ptr, d_src.ptr if d_src else None, plane.strides[0], None))
        device.sync()
        return d_pl.download(np.uint16, plane.shape)

    def run_dc(c422, recs, coeffs, luma_dc):
        d_rec, d_co, d_dc = _dev(recs), _dev(coeffs), _dev(luma_dc)
        gpu.check(lib.ff_h264_dc_dequant_batch_hbd_cuda(1 + c422, d_rec.ptr, recs.shape[0], d_co.ptr, 768, d_dc.ptr, None))
        device.sync()
        return d_co.download(np.int32, coeffs.shape)
    hh.weight_dc_cases(run_weight, run_dc, checker, bits)


@pytest.mark.parametrize("bits", [9, 10])
@pytest.mark.parametrize("mb_w,mb_h,P,p_intra", [(3, 2, 1, 1.0), (7, 5, 2, 1.0), (20, 12, 2, 0.6), (40, 30, 3, 1.0)])
def test_intra_batch_hbd(gpu, checker, mb_w, mb_h, P, p_intra, bits):
    """ff_h264_intra_mb_batch_hbd_cuda: all-intra and mixed pictures, stacked; samples and consumed coefficients against the oracle chain"""
    from libav_b200 import device
    ys, cbs, crs, recs, cos, nzs, want = [], [], [], [], [], [], []
    for k in range(P):
        y, cb, cr = hh.picture(mb_w, mb_h, bits, 0, seed=50 + k)
        rec, coeffs, nnzc = hh.intra_work(mb_w, mb_h, bits, seed=mb_w + k, p_intra=p_intra)
        wy, wcb, wcr, wco = y.copy(), cb.copy(), cr.copy(), coeffs.copy()
        hh.oracle_intra(checker, bits, rec, wco, nnzc, mb_w, mb_h, wy, wcb, wcr)
        assert not np.array_equal(wy, y)
        ys.append(y); cbs.append(cb); crs.append(cr); recs.append(rec); cos.append(coeffs); nzs.append(nnzc); want.append((wy, wcb, wcr, wco))
    Y, CB, CR = np.concatenate(ys), np.concatenate(cbs), np.concatenate(crs)
    R, CO, NZ = np.concatenate(recs), np.concatenate(cos), np.concatenate(nzs)
    d_rec, d_co, d_nz, dy, dcb, dcr = _dev(R), _dev(CO), _dev(NZ), _dev(Y), _dev(CB), _dev(CR)
    gpu.check(gpu.lib.ff_h264_intra_mb_batch_hbd_cuda(bits, d_rec.ptr, mb_w, mb_h, P, d_co.ptr, 768, d_nz.ptr, dy.ptr, dcb.ptr, dcr.ptr, Y.strides[0], CB.strides[0], None))
    device.sync()
    gy, gcb, gcr, gco = dy.download(np.uint16, Y.shape), dcb.download(np.uint16, CB.shape), dcr.download(np.uint16, CR.shape), d_co.download(np.int32, CO.shape)
    n = mb_w * mb_h
    for k in range(P):
        assert np.array_equal(gy[16 * mb_h * k:16 * mb_h * (k + 1)], want[k][0]), (k, np.argwhere(gy[16 * mb_h * k:16 * mb_h * (k + 1)] != want[k][0])[:4].tolist())
        assert np.array_equal(gcb[8 * mb_h * k:8 * mb_h * (k + 1)], want[k][1]) and np.array_equal(gcr[8 * mb_h * k:8 * mb_h * (k + 1)], want[k][2]), k
        assert np.array_equal(gco[n * k:n * (k + 1)], want[k][3]), k


@pytest.mark.parametrize("bits", [9, 10])
@pytest.mark.parametrize("mb_w,mb_h,P,p_intra", [(7, 5, 1, 0.3), (20, 12, 2, 0.25)])
def test_flush_hbd_decides_at_the_streams_bit_depth(gpu, checker, mb_w, mb_h, P, p_intra, bits):
    """ff_h264_flush_pictures_cuda with bit_depth 9 / 10: MC -> weighted prediction -> DC transforms -> residual -> intra -> decisions -> loop filter in one
    call, against the CPU checker's BIT_DEPTH > 8 functions chained in the same order on the same records; the checker decides at the stream's
    bit depth"""
    import ctypes as C
    from libav_b200 import device, tables
    from oracle.loader import ptr
    from test_gpu_h264flush import picture_work
    from test_oracle_h264lf_hbd_cpu import hbd_oracle, run as oracle_decisions
    sc = 1 << (bits - 8)
    refs = [hh.picture(mb_w, mb_h, bits, 0, seed=11), hh.picture(mb_w, mb_h, bits, 0, seed=12)]
    works = [picture_work(mb_w, mb_h, 100 * k + mb_w, p_intra) for k in range(P)]
    for w in works:         # the side information a 9 / 10-bit decoder keeps: qscale_table, chroma_qp_table and qp_thresh in the QP' scale
        w["info"] = synth.h264_deblock_info(mb_w, mb_h, seed=mb_w + 4, n_slices=3, bipred=True, t8x8=1, cabac=1, bit_depth=bits)
    pics = [hh.picture(mb_w, mb_h, bits, 0, seed=50 + k) for k in range(P)]
    ls, uvls = pics[0][0].strides[0], pics[0][1].strides[0]
    want, want_co = [], []
    for w, (y, cb, cr) in zip(works, pics):
        w["coeffs"] = w["coeffs"].astype(np.int32) * sc
        w["luma_dc"] = w["luma_dc"].astype(np.int32) * sc
        w["res"]["luma_off"] *= 2; w["res"]["chroma_off"] *= 2; w["weight"]["off"] *= 2       # byte offsets for 16-bit samples
        wy, wcb, wcr = y.copy(), cb.copy(), cr.copy()
        hh.oracle_mc(checker, bits, 0, w["mc"], refs, wy, wcb, wcr)
        for r in w["weight"]:
            checker.h264_hbd_weight(bits, 0, hh.at(wy, r["off"]), ls, int(r["h"]), int(r["log2_denom"]), int(r["weight"]), int(r["offset"]))
        co = w["coeffs"].copy()
        for m in range(co.shape[0]):
            if w["dc"]["luma_qmul"][m]:
                checker.h264_hbd_dc_dequant(bits, 0, hh.at(co, m * 768 * 4), ptr(w["luma_dc"][m].copy()), int(w["dc"]["luma_qmul"][m]))
            for p in range(2):
                if w["dc"]["chroma_qmul"][m, p]:
                    checker.h264_hbd_dc_dequant(bits, 1, hh.at(co, (m * 768 + 256 * (p + 1)) * 4), None, int(w["dc"]["chroma_qmul"][m, p]))
        hh.oracle_residual(checker, bits, 0, w["res"], co, w["nnzc"], wy, wcb, wcr)
        hh.oracle_intra(checker, bits, w["intra"], co, w["nnzc"], mb_w, mb_h, wy, wcb, wcr)
        rec = oracle_decisions(hbd_oracle(checker), w["info"]).view(synth.DEBLOCK_DT).reshape(-1)
        hh.oracle_deblock(checker, bits, rec, mb_w, mb_h, wy, wcb, wcr)
        want.append((wy, wcb, wcr)); want_co.append(co)
    Y, CB, CR = (np.concatenate([p[i] for p in pics]) for i in range(3))
    cat = lambda k: np.concatenate([w[k] for w in works])
    mc, res, wrec = [], [], []
    for k, w in enumerate(works):
        m = w["mc"].copy(); m["y"] += 16 * mb_h * k; mc.append(m)
        r = w["res"].copy(); r["luma_off"] += 16 * mb_h * k * ls; r["chroma_off"] += 8 * mb_h * k * uvls; res.append(r)
        t = w["weight"].copy(); t["off"] += 16 * mb_h * k * ls; wrec.append(t)
    mc, res, wrec = np.concatenate(mc), np.concatenate(res), np.concatenate(wrec)
    mc = np.concatenate([mc[mc["avg"] == 0], mc[mc["avg"] != 0]])
    dref = [[_dev(np.concatenate([p] * P)) for p in r] for r in refs]
    d_planes = _dev(np.array([[p.ptr for p in r] for r in dref], dtype=np.uint64))
    infos = [w["info"] for w in works]
    catinfo = lambda k: np.concatenate([d[k] for d in infos], axis=0)
    keep = {k: _dev(catinfo(k)) for k in ("mb_type", "qscale", "nnz", "cbp", "slice_table", "mv0", "mv1", "ref0", "ref1")}
    keep["sp"] = _dev(infos[0]["slice_params"]); keep["cq"] = _dev(infos[0]["chroma_qp_table"])
    info = tables.FFH264DeblockInfo(mb_w, mb_h, P, keep["mb_type"].ptr, keep["qscale"].ptr, keep["nnz"].ptr, keep["cbp"].ptr, keep["slice_table"].ptr,
                                    (C.c_void_p * 2)(keep["mv0"].ptr, keep["mv1"].ptr), (C.c_void_p * 2)(keep["ref0"].ptr, keep["ref1"].ptr),
                                    keep["sp"].ptr, infos[0]["n_slices"], keep["cq"].ptr, infos[0]["cabac"], infos[0]["t8x8"])
    n = mb_w * mb_h * P
    d = dict(y=_dev(Y), cb=_dev(CB), cr=_dev(CR), mc=_dev(mc), res=_dev(res), w=_dev(wrec), co=_dev(cat("coeffs")), nz=_dev(cat("nnzc")),
             dc=_dev(cat("dc")), ldc=_dev(cat("luma_dc")), intra=_dev(cat("intra")), rec=device.DevBuf(n * 104))
    work = tables.FFH264PictureWork()
    work.mb_w, work.mb_h, work.n_pictures = mb_w, mb_h, P
    work.luma, work.cb, work.cr, work.linesize, work.uvlinesize = d["y"].ptr, d["cb"].ptr, d["cr"].ptr, ls, uvls
    work.mc, work.n_mc, work.refs = d["mc"].ptr, mc.shape[0], d_planes.ptr
    work.weight[0], work.n_weight[0] = d["w"].ptr, wrec.shape[0]
    work.coeffs, work.coeff_stride, work.nnzc = d["co"].ptr, 768, d["nz"].ptr
    work.dc, work.luma_dc, work.residual, work.intra = d["dc"].ptr, d["ldc"].ptr, d["res"].ptr, d["intra"].ptr
    work.deblock_info, work.deblock_records = C.pointer(info), d["rec"].ptr
    work.bit_depth, work.chroma_format_idc = bits, 1
    gpu.check(gpu.lib.ff_h264_flush_pictures_cuda(C.byref(work), None))
    device.sync()
    gy, gcb, gcr = d["y"].download(np.uint16, Y.shape), d["cb"].download(np.uint16, CB.shape), d["cr"].download(np.uint16, CR.shape)
    wy = np.concatenate([w[0] for w in want])
    assert np.array_equal(gy, wy), np.argwhere(gy != wy)[:5].tolist()
    assert np.array_equal(gcb, np.concatenate([w[1] for w in want])) and np.array_equal(gcr, np.concatenate([w[2] for w in want]))
    assert np.array_equal(d["co"].download(np.int32, (n, 768)), np.concatenate(want_co))


def test_dc_dequant_batch_422_8bit(gpu, checker):
    """ff_h264_dc_dequant_batch_422_cuda: int16 coefficients, the 2 x 4 chroma DC transform of chroma_format_idc 2 (h264idct_template.c:271-306)"""
    from libav_b200 import device
    from oracle.loader import ptr
    rng = np.random.default_rng(422)
    n = 300
    recs = np.zeros(n, np.dtype([("luma_qmul", "<u4"), ("chroma_qmul", "<u4", (2,))]))
    recs["luma_qmul"] = np.where(rng.random(n) < 0.6, rng.integers(16, 1200, n), 0)
    recs["chroma_qmul"] = np.where(rng.random((n, 2)) < 0.6, rng.integers(16, 1200, (n, 2)), 0)
    coeffs = rng.integers(-120, 120, size=(n, 768)).astype(np.int16)
    luma_dc = rng.integers(-500, 500, size=(n, 16)).astype(np.int16)
    want = coeffs.copy()
    for m in range(n):
        if recs["luma_qmul"][m]:
            checker.h264_luma_dc_dequant_idct(hh.at(want, m * 768 * 2), ptr(luma_dc[m].copy()), int(recs["luma_qmul"][m]))
        for pl in range(2):
            if recs["chroma_qmul"][m, pl]:
                checker.h264_chroma422_dc_dequant_idct(hh.at(want, (m * 768 + 256 * (pl + 1)) * 2), int(recs["chroma_qmul"][m, pl]))
    d_rec, d_co, d_dc = _dev(recs), _dev(coeffs), _dev(luma_dc)
    gpu.check(gpu.lib.ff_h264_dc_dequant_batch_422_cuda(d_rec.ptr, n, d_co.ptr, 768, d_dc.ptr, None))
    device.sync()
    got = d_co.download(np.int16, coeffs.shape)
    assert not np.array_equal(want, coeffs) and np.array_equal(got, want), np.argwhere(got != want)[:4].tolist()


@pytest.mark.parametrize("bits", [8, 10])
@pytest.mark.parametrize("mb_w,mb_h,P,p_intra", [(7, 5, 1, 0.0), (20, 12, 2, 0.3)])
def test_flush_422_pictures(gpu, checker, mb_w, mb_h, P, p_intra, bits):
    """ff_h264_flush_pictures_cuda with chroma_format_idc 2 (8 and 10 bit), caller-filled deblocking records: MC -> weighted prediction -> DC transforms
    (2 x 4 chroma) -> residual -> intra macroblocks (8 x 16 chroma predictors) -> 4:2:2 loop filter in one call, against the CPU checker chained
    in the same order"""
    flush_422(gpu, checker, mb_w, mb_h, P, p_intra, bits)


def flush_422(gpu, checker, mb_w, mb_h, P, p_intra, bits, decide=False):
    """decide: the flush derives the deblocking records from FFH264DeblockInfo (side information in the decoder's scale for `bits`, the
    chroma422 array of the decisions); the checker decides at `bits` and both sets of records are compared as well as the pictures"""
    import ctypes as C
    from libav_b200 import device, tables
    from oracle.loader import ptr
    from test_oracle_h264lf_hbd_cpu import hbd_oracle, run422
    from test_gpu_h264lf import device_info
    sb = 1 if bits == 8 else 2
    cdt = np.int16 if bits == 8 else np.int32
    rng = np.random.default_rng(bits * 100 + mb_w)
    refs = [hh.smooth_picture422(mb_w, mb_h, bits, seed=11), hh.smooth_picture422(mb_w, mb_h, bits, seed=12)]
    n1 = mb_w * mb_h
    pics, mcs, ress, cos, nzs, dcs, wrecs, recs, exts, want, want_co, irecs = [], [], [], [], [], [], [], [], [], [], [], []
    if decide:
        infos = [synth.h264_deblock_info(mb_w, mb_h, seed=60 + k, n_slices=3, bipred=True, t8x8=1, bit_depth=bits) for k in range(P)]
        for d_ in infos[1:]:                                                   # one set of slice headers / PPS per flush
            d_["slice_params"], d_["chroma_qp_table"] = infos[0]["slice_params"], infos[0]["chroma_qp_table"]
    for k in range(P):
        y, cb, cr = hh.smooth_picture422(mb_w, mb_h, bits, seed=50 + k)
        ls, uvls = y.strides[0], cb.strides[0]
        mc = synth.h264_mc_work(mb_w, mb_h, seed=mb_h + k, max_mv=24, avg_second=True)
        res, co, nz = hh.residual_work(mb_w, mb_h, bits, 1, y, cb, seed=mb_w + k)
        co = (co // 4).astype(cdt)                                             # small residual: the loop filter still has edges to change
        irec, ico, inz = hh.intra_work(mb_w, mb_h, bits, seed=31 + k, p_intra=p_intra, c422=1)
        intra = irec["kind"] != 0                                              # intra macroblocks: no MC / weight / inter residual, their own coefficients
        res["luma_mode"][intra] = 3; res["chroma"][intra] = 0
        co[intra] = ico[intra]; nz[intra] = inz[intra]
        mc = mc[~intra[(mc["y"] // 16) * mb_w + mc["x"] // 16]]
        dc = np.zeros(n1, np.dtype([("luma_qmul", "<u4"), ("chroma_qmul", "<u4", (2,))]))
        dc["chroma_qmul"] = np.where(rng.random((n1, 2)) < 0.5, rng.integers(16, 200, (n1, 2)), 0)
        wr = []
        for m in range(n1):
            if rng.random() < 0.4 and not intra[m]:
                wr.append(((m // mb_w) * 16 * ls + (m % mb_w) * 16 * sb, 16, 16, int(rng.integers(0, 7)), 0, int(rng.integers(-20, 90)), 0, int(rng.integers(-20, 20)), 0))
        wr = np.array(wr, dtype=synth.WEIGHT_DT)
        if decide:
            rec, ext = run422(hbd_oracle(checker), infos[k])
            rec, ext = rec.view(synth.DEBLOCK_DT).reshape(-1), ext.view(hh.CHROMA422_DT).reshape(-1)
        else:
            rec, ext = hh.deblock422_work(mb_w, mb_h, seed=3 + k, slices=2)
        wy, wcb, wcr, wco = y.copy(), cb.copy(), cr.copy(), co.copy()
        hh.oracle_mc(checker, bits, 1, mc, refs, wy, wcb, wcr)
        for r in wr:
            if bits == 8:
                checker.h264_weight(0, hh.at(wy, r["off"]), ls, int(r["h"]), int(r["log2_denom"]), int(r["weight"]), int(r["offset"]))
            else:
                checker.h264_hbd_weight(bits, 0, hh.at(wy, r["off"]), ls, int(r["h"]), int(r["log2_denom"]), int(r["weight"]), int(r["offset"]))
        for m in range(n1):
            for p in range(2):
                if dc["chroma_qmul"][m, p]:
                    o_ = (m * 768 + 256 * (p + 1)) * wco.itemsize
                    if bits == 8:
                        checker.h264_chroma422_dc_dequant_idct(hh.at(wco, o_), int(dc["chroma_qmul"][m, p]))
                    else:
                        checker.h264_hbd_dc_dequant(bits, 2, hh.at(wco, o_), None, int(dc["chroma_qmul"][m, p]))
        hh.oracle_residual(checker, bits, 1, res, wco, nz, wy, wcb, wcr)
        hh.oracle_intra(checker, bits, irec, wco, nz, mb_w, mb_h, wy, wcb, wcr, c422=1)
        pre = wy.copy()
        hh.oracle_deblock422(checker, bits, rec, ext, mb_w, mb_h, wy, wcb, wcr)
        assert not np.array_equal(pre, wy)
        m2 = mc.copy(); m2["y"] += 16 * mb_h * k
        r2 = res.copy(); r2["luma_off"] += 16 * mb_h * k * ls; r2["chroma_off"] += 16 * mb_h * k * uvls
        w2 = wr.copy(); w2["off"] += 16 * mb_h * k * ls
        pics.append((y, cb, cr)); mcs.append(m2); ress.append(r2); cos.append(co); nzs.append(nz); dcs.append(dc); wrecs.append(w2); irecs.append(irec)
        recs.append(rec); exts.append(ext); want.append((wy, wcb, wcr)); want_co.append(wco)
    Y, CB, CR = (np.concatenate([p[i] for p in pics]) for i in range(3))
    mc = np.concatenate(mcs)
    mc = np.concatenate([mc[mc["avg"] == 0], mc[mc["avg"] != 0]])
    wrec = np.concatenate(wrecs)
    dref = [[_dev(np.concatenate([p] * P)) for p in r] for r in refs]
    d_planes = _dev(np.array([[p.ptr for p in r] for r in dref], dtype=np.uint64))
    n = n1 * P
    d = dict(y=_dev(Y), cb=_dev(CB), cr=_dev(CR), mc=_dev(mc), res=_dev(np.concatenate(ress)), w=_dev(wrec), co=_dev(np.concatenate(cos)),
             nz=_dev(np.concatenate(nzs)), dc=_dev(np.concatenate(dcs)), ldc=_dev(np.zeros((n, 16), cdt)), rec=_dev(np.concatenate(recs)),
             ext=_dev(np.concatenate(exts)), intra=_dev(np.concatenate(irecs)))
    work = tables.FFH264PictureWork()
    work.mb_w, work.mb_h, work.n_pictures = mb_w, mb_h, P
    work.luma, work.cb, work.cr, work.linesize, work.uvlinesize = d["y"].ptr, d["cb"].ptr, d["cr"].ptr, Y.strides[0], CB.strides[0]
    work.mc, work.n_mc, work.refs = d["mc"].ptr, mc.shape[0], d_planes.ptr
    work.weight[0], work.n_weight[0] = d["w"].ptr, wrec.shape[0]
    work.coeffs, work.coeff_stride, work.nnzc = d["co"].ptr, 768, d["nz"].ptr
    work.dc, work.luma_dc, work.residual = d["dc"].ptr, d["ldc"].ptr, d["res"].ptr
    if p_intra:
        work.intra = d["intra"].ptr
    if decide:
        d["rec"].fill(0xAB); d["ext"].fill(0xCD)
        info, keep = device_info(infos, chroma422=d["ext"].ptr)
        work.deblock_info, work.deblock_records = C.pointer(info), d["rec"].ptr
    else:
        work.deblock_records, work.deblock_chroma422 = d["rec"].ptr, d["ext"].ptr
    work.bit_depth, work.chroma_format_idc = bits, 2
    gpu.check(gpu.lib.ff_h264_flush_pictures_cuda(C.byref(work), None))
    device.sync()
    if decide:
        assert np.array_equal(d["rec"].download(np.uint8, (n, 104)), np.concatenate(recs).view(np.uint8).reshape(n, 104))
        assert np.array_equal(d["ext"].download(np.uint8, (n, 52)), np.concatenate(exts).view(np.uint8).reshape(n, 52))
    gy, gcb, gcr = d["y"].download(Y.dtype, Y.shape), d["cb"].download(Y.dtype, CB.shape), d["cr"].download(Y.dtype, CR.shape)
    wy = np.concatenate([w[0] for w in want])
    assert np.array_equal(gy, wy), np.argwhere(gy != wy)[:5].tolist()
    assert np.array_equal(gcb, np.concatenate([w[1] for w in want])) and np.array_equal(gcr, np.concatenate([w[2] for w in want]))
    assert np.array_equal(d["co"].download(cdt, (n, 768)), np.concatenate(want_co))


@pytest.mark.parametrize("bits", [8, 9, 10])
@pytest.mark.parametrize("mb_w,mb_h,P,p_intra", [(3, 2, 1, 1.0), (7, 5, 2, 1.0), (20, 12, 2, 0.6), (40, 30, 3, 1.0)])
def test_intra_batch_422(gpu, checker, mb_w, mb_h, P, p_intra, bits):
    """ff_h264_intra_mb_batch_422_cuda: 8 x 16 chroma predictors + h264_idct_add8_422, 8-bit (uint8 / int16) and 9 / 10-bit (uint16 / int32) pictures, stacked"""
    from libav_b200 import device
    ys, cbs, crs, recs, cos, nzs, want = [], [], [], [], [], [], []
    for k in range(P):
        y, cb, cr = hh.picture(mb_w, mb_h, bits, 1, seed=50 + k)
        rec, coeffs, nnzc = hh.intra_work(mb_w, mb_h, bits, seed=mb_w + k, p_intra=p_intra, c422=1)
        wy, wcb, wcr, wco = y.copy(), cb.copy(), cr.copy(), coeffs.copy()
        hh.oracle_intra(checker, bits, rec, wco, nnzc, mb_w, mb_h, wy, wcb, wcr, c422=1)
        assert not np.array_equal(wy, y) and not np.array_equal(wcb, cb)
        ys.append(y); cbs.append(cb); crs.append(cr); recs.append(rec); cos.append(coeffs); nzs.append(nnzc); want.append((wy, wcb, wcr, wco))
    Y, CB, CR = np.concatenate(ys), np.concatenate(cbs), np.concatenate(crs)
    R, CO, NZ = np.concatenate(recs), np.concatenate(cos), np.concatenate(nzs)
    d_rec, d_co, d_nz, dy, dcb, dcr = _dev(R), _dev(CO), _dev(NZ), _dev(Y), _dev(CB), _dev(CR)
    gpu.check(gpu.lib.ff_h264_intra_mb_batch_422_cuda(bits, d_rec.ptr, mb_w, mb_h, P, d_co.ptr, 768, d_nz.ptr, dy.ptr, dcb.ptr, dcr.ptr, Y.strides[0], CB.strides[0], None))
    device.sync()
    gy, gcb, gcr, gco = dy.download(Y.dtype, Y.shape), dcb.download(Y.dtype, CB.shape), dcr.download(Y.dtype, CR.shape), d_co.download(CO.dtype, CO.shape)
    n, H = mb_w * mb_h, 16 * mb_h
    for k in range(P):
        assert np.array_equal(gy[H * k:H * (k + 1)], want[k][0]), (k, np.argwhere(gy[H * k:H * (k + 1)] != want[k][0])[:4].tolist())
        assert np.array_equal(gcb[H * k:H * (k + 1)], want[k][1]), (k, np.argwhere(gcb[H * k:H * (k + 1)] != want[k][1])[:4].tolist())
        assert np.array_equal(gcr[H * k:H * (k + 1)], want[k][2]), k
        assert np.array_equal(gco[n * k:n * (k + 1)], want[k][3]), k
