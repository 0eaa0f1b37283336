"""The edge cases of tests/h264_edge_cases.py at 9 / 10 bit and in 4:2:2 on the CPU: the batched calls of h264_hbd_batch.cu that
tests/hostsim/ compiles as host C++ -- residual, MC (its clamped-global-load form), weighted prediction, DC transforms -- against the
checker (the compiled reference where it is built, else the port) on decoder-layout pictures inside poisoned allocations: far, limit
and outside vectors, pictures stacked in one call, shuffled records, coefficients at both ends of the legal range, every dispatch rule,
every weight corner, and the misaligned arguments the 16-bit calls refuse.  The port is pinned to the reference on the same cases.
The GPU runs them through the device kernels, the staged MC and the deblocking wavefront as well (tests/test_gpu_h264_hbd_edges.py)."""
import numpy as np
import pytest

import h264_edge_cases as ec
import h264_hbd_util as hh
import hostsim_build

MB_W, MB_H = 12, 8
TIGHT = ec.Layout("tight", 0, 0)
CASES = [(9, 0), (9, 1), (10, 0), (10, 1), (8, 1)]            # (bits, 4:2:2); 8-bit 4:2:2 where the call takes it
case_id = lambda c: "%dbit-%s" % (c[0], "422" if c[1] else "420")
MC_LAYOUTS = [TIGHT, *ec.HBD_LAYOUTS, ec.REF2]
REFUSED = [ec.SHIFT1, ec.ODD_CB, ec.ODD_UV, ec.ODD_LS]


@pytest.fixture(scope="module")
def sim(built):
    return hostsim_build.fresh()


def place_all(lay, planes, ref=False):
    return [lay.place(p, chroma=i > 0, ref=ref) for i, p in enumerate(planes)]


def check_all(placed, want, what=""):
    for (b, v), w, name in zip(placed, want, ("y", "cb", "cr")):
        ec.Layout.check(b, v, w, (what, name))


# ---- motion compensation ----
def mc_case(o, bits, c422, seed, mb_w=MB_W, mb_h=MB_H, band=34):
    refs = [hh.picture(mb_w, mb_h, bits, c422, seed=seed + k) for k in range(2)]
    dst = hh.picture(mb_w, mb_h, bits, c422, seed=seed + 2)
    rec = ec.mc_records(mb_w, mb_h, seed=seed + 3, band=band)
    return refs, dst, rec, oracle_mc(o, bits, c422, rec, refs, dst)


def oracle_mc(o, bits, c422, rec, refs, dst):
    want = [p.copy() for p in dst]
    hh.oracle_mc(o, bits, c422, rec, refs, *want)
    return want


def sim_mc(lib, bits, c422, rec, refs, dst, lay, pw, ph):
    d = place_all(lay, dst)
    r = [place_all(lay, rp, ref=True) for rp in refs]
    planes = np.array([[v.ctypes.data for _, v in rp] for rp in r], np.uint64)
    assert lib.ff_h264_mc_batch_hbd_cuda(bits, 1 + c422, rec.ctypes.data, rec.shape[0], planes.ctypes.data, *(v.ctypes.data for _, v in d),
                                         d[0][1].strides[0], d[1][1].strides[0], pw, ph, None) == 0
    for rp, want in zip(r, refs):
        check_all(rp, want, "reference")
    return d


@pytest.fixture(scope="module", params=CASES, ids=case_id)
def mc_far(request, checker):
    bits, c422 = request.param
    return (bits, c422) + mc_case(checker, bits, c422, seed=40 + bits + 5 * c422)


@pytest.mark.parametrize("lay", MC_LAYOUTS, ids=repr)
def test_mc_far_vectors_in_decoder_layout(sim, mc_far, lay):
    bits, c422, refs, dst, rec, want = mc_far
    check_all(sim_mc(sim, bits, c422, rec, refs, dst, lay, 16 * MB_W, 16 * MB_H), want, lay)


def test_mc_any_record_order_and_batch_size(sim, checker, mc_far):
    """put and avg records interleaved in any order, batch sizes that are not multiples of the four records of a thread block"""
    bits, c422, refs, dst, rec, want = mc_far
    perm = rec[np.random.default_rng(5).permutation(rec.shape[0])]
    assert any(perm["avg"][k] and not perm["avg"][k + 1] for k in range(perm.shape[0] - 1))
    check_all(sim_mc(sim, bits, c422, perm, refs, dst, ec.PAD2, 16 * MB_W, 16 * MB_H), want, "permuted")
    for n in (1, 7, 33, 130):
        sub = perm[:n]
        check_all(sim_mc(sim, bits, c422, sub, refs, dst, ec.PAD2, 16 * MB_W, 16 * MB_H), oracle_mc(checker, bits, c422, sub, refs, dst), n)


def stacked_mc_case(o, bits, c422, P):
    """P pictures stacked in the same planes with far vectors: each record's fetches clamp to its own picture's rows"""
    mb_w, mb_h = 6, 4
    H = 16 * mb_h
    cases = [mc_case(o, bits, c422, seed=90 + 10 * k, mb_w=mb_w, mb_h=mb_h, band=0) for k in range(P)]
    cat = lambda planes: [np.concatenate([p[i] for p in planes]) for i in range(3)]
    recs = []
    for k, c in enumerate(cases):
        r = c[2].copy(); r["y"] += k * H; recs.append(r)
    refs = [cat([c[0][j] for c in cases]) for j in range(2)]
    # vectors that would cross a seam: the oracle of each picture sees only its own rows, the stacked planes hold the neighbours
    crossing = sum(int(((c[2]["mvy"] + 4 * c[2]["y"]) >> 2 < -2).sum() + ((c[2]["mvy"] + 4 * c[2]["y"]) >> 2 > H + 2).sum()) for c in cases)
    assert crossing > 20, crossing
    return np.concatenate(recs), refs, cat([c[1] for c in cases]), cat([c[3] for c in cases]), mb_w, H


@pytest.mark.parametrize("P", [2, 3])
@pytest.mark.parametrize("case", CASES, ids=case_id)
def test_mc_stacked_pictures_far_vectors(sim, checker, case, P):
    bits, c422 = case
    rec, refs, dst, want, mb_w, H = stacked_mc_case(checker, bits, c422, P)
    check_all(sim_mc(sim, bits, c422, rec, refs, dst, ec.PAD4, 16 * mb_w, H), want)


# ---- residual ----
def residual_case(o, bits, c422, seed, mb_w=9, mb_h=6):
    rec, coeffs, nnzc = ec.residual_records(mb_w, mb_h, seed=seed, bits=bits, c422=c422)
    pic = hh.picture(mb_w, mb_h, bits, c422, seed=seed + 1)
    want, want_co = [p.copy() for p in pic], coeffs.copy()
    hh.oracle_residual(o, bits, c422, rec, want_co, nnzc, *want)
    top = (1 << bits) - 1
    for p, w in zip(pic, want):                                         # the destination clips at both ends
        assert ((w == 0) & (p != 0)).any() and ((w == top) & (p != top)).any()
    return mb_w, rec, coeffs, nnzc, pic, want, want_co


def run_residual(call, bits, c422, case, lay, stride):
    """the call on the picture placed by `lay` and an arena of `stride` coefficients per macroblock whose tail is poisoned; checks the
    pixels, the consumed arena and every poisoned byte"""
    mb_w, rec, coeffs, nnzc, pic, want, want_co = case
    n, sb = coeffs.shape[0], pic[0].itemsize
    d = place_all(lay, pic)
    r2 = ec.relayout_residual(rec, 16 * mb_w * sb, d[0][1].strides[0], d[1][1].strides[0])
    arena = np.full((n, stride), -0x5A5A5A5B, coeffs.dtype) if sb == 2 else np.full((n, stride), 0x5A5A, coeffs.dtype)
    poison = arena[0, -1]
    arena[:, :768] = coeffs
    assert call(bits, 1 + c422, r2, arena, stride, nnzc, d) == 0
    check_all(d, want)
    assert np.array_equal(arena[:, :768], want_co), np.argwhere(arena[:, :768] != want_co)[:5].tolist()
    assert (arena[:, 768:] == poison).all()
    assert (want_co != 0).any()                                         # blocks the dispatchers skip, and AC left behind, stay


def sim_residual(lib):
    return lambda bits, idc, rec, arena, stride, nnzc, d: lib.ff_h264_idct_add_mb_batch_hbd_cuda(
        bits, idc, rec.ctypes.data, rec.shape[0], arena.ctypes.data, stride, nnzc.ctypes.data, *(v.ctypes.data for _, v in d),
        d[0][1].strides[0], d[1][1].strides[0], None)


@pytest.fixture(scope="module", params=CASES, ids=case_id)
def res_case(request, checker):
    bits, c422 = request.param
    return (bits, c422, residual_case(checker, bits, c422, seed=61 + bits + 3 * c422))


@pytest.mark.parametrize("lay,stride", [(TIGHT, 768), (ec.PAD4, 776), (ec.PAD2, 768), (ec.SHIFT2, 768), (ec.CSHIFT2, 770)],
                         ids=lambda v: repr(v))
def test_residual_range_ends_and_dispatch(sim, res_case, lay, stride):
    bits, c422, case = res_case
    run_residual(sim_residual(sim), bits, c422, case, lay, stride)


# ---- weighted prediction and DC transforms ----
def weight_case(o, bits, bi, seed):
    rec, plane, src = ec.weight_records(bi, seed=seed, bits=bits)
    want = plane.copy()
    hh.oracle_weight(o, bits, rec, want, src if bi else None)
    top = (1 << bits) - 1
    assert ((want == 0) & (plane != 0)).any() and ((want == top) & (plane != top)).any()       # clipped at both ends
    return rec, plane, src, want


def run_weight(call, bits, bi, case, lay):
    rec, plane, src, want = case
    lp, ls_ = lay.place(plane), lay.place(src)
    ls = lp[1].strides[0]
    r2 = rec.copy(); r2["off"] = ec.relayout_offsets(rec["off"], plane.shape[1] * plane.itemsize, ls)
    assert call(bits, r2, lp, ls_ if bi else None, ls) == 0
    ec.Layout.check(*lp, want)
    ec.Layout.check(*ls_, src, "second prediction")


def sim_weight(lib):
    return lambda bits, rec, lp, ls_, ls: lib.ff_h264_weight_batch_hbd_cuda(bits, rec.ctypes.data, rec.shape[0], lp[1].ctypes.data,
                                                                             ls_[1].ctypes.data if ls_ else None, ls, None)


@pytest.mark.parametrize("lay", [TIGHT, ec.PAD2, ec.SHIFT2], ids=repr)
@pytest.mark.parametrize("bi", [0, 1])
@pytest.mark.parametrize("bits", [9, 10])
def test_weight_every_corner(sim, checker, bits, bi, lay):
    run_weight(sim_weight(sim), bits, bi, weight_case(checker, bits, bi, seed=43 + bi), lay)


def dc_case(o, bits, c422, seed):
    rec, coeffs, luma_dc = ec.dc_records(300, bits, c422, seed)
    want = coeffs.copy()
    hh.oracle_dc(o, bits, c422, rec, want, luma_dc)
    return rec, coeffs, luma_dc, want


def run_dc(call, c422, case, stride=776):
    rec, coeffs, luma_dc, want = case
    arena = np.full((coeffs.shape[0], stride), -0x5A5A5A5B, np.int32)
    arena[:, :768] = coeffs
    assert call(1 + c422, rec, arena, stride, luma_dc) == 0
    assert np.array_equal(arena[:, :768], want), np.argwhere(arena[:, :768] != want)[:5].tolist()
    assert (arena[:, 768:] == -0x5A5A5A5B).all()


@pytest.mark.parametrize("c422", [0, 1])
@pytest.mark.parametrize("bits", [9, 10])
def test_dc_range_ends_and_largest_qmul(sim, checker, bits, c422):
    call = lambda idc, rec, arena, stride, luma_dc: sim.ff_h264_dc_dequant_batch_hbd_cuda(idc, rec.ctypes.data, rec.shape[0], arena.ctypes.data, stride,
                                                                                         luma_dc.ctypes.data, None)
    run_dc(call, c422, dc_case(checker, bits, c422, seed=7 + bits + c422))


# ---- refusals ----
@pytest.mark.parametrize("lay", REFUSED, ids=repr)
def test_refuses_odd_planes_and_pitches(sim, lay):
    """16-bit samples at an odd address or with an odd pitch: -1, the error message, and not one byte written"""
    pic = hh.picture(2, 2, 10, 1, seed=3)
    d = place_all(lay, pic)
    ptrs, ls, uvls = [v.ctypes.data for _, v in d], d[0][1].strides[0], d[1][1].strides[0]
    rec = ec.mc_records(12, 8, seed=1)[:8]
    planes = np.array([ptrs] * 2, np.uint64)
    res = np.zeros(4, ec.synth.RESIDUAL_DT)
    co, nz = np.ones((4, 768), np.int32), np.full((4, 120), 3, np.uint8)
    wrec = np.zeros(1, ec.synth.WEIGHT_DT); wrec["w"] = wrec["h"] = 8; wrec["weight"] = 3
    odd = 0 if (ls | ptrs[0]) & 1 else 1                                # the plane (and pitch) a weight call would take
    calls = [lambda: sim.ff_h264_mc_batch_hbd_cuda(10, 2, rec.ctypes.data, rec.shape[0], planes.ctypes.data, *ptrs, ls, uvls, 32, 32, None),
             lambda: sim.ff_h264_idct_add_mb_batch_hbd_cuda(10, 2, res.ctypes.data, 4, co.ctypes.data, 768, nz.ctypes.data, *ptrs, ls, uvls, None),
             lambda: sim.ff_h264_weight_batch_hbd_cuda(10, wrec.ctypes.data, 1, ptrs[odd], None, (ls, uvls)[odd], None)]
    for k, call in enumerate(calls):
        assert call() == -1, k
        assert "16-bit samples need even plane addresses and pitches" in sim.avb200_last_error().decode(), k
        sim.avb200_clear_error()
    check_all(d, pic)
    assert (co == 1).all()


# ---- the port as a checker ----
def test_port_pinned_to_reference(orc, refo):
    """the port's 9 / 10-bit and 4:2:2 functions against the reference on these generators: MC (far vectors), residual (range ends),
    weights (every corner), DC transforms and the loop filters (high qp on blocky content)"""
    for bits, c422 in CASES:
        a, b = mc_case(orc, bits, c422, seed=5, mb_w=6, mb_h=4, band=0), mc_case(refo, bits, c422, seed=5, mb_w=6, mb_h=4, band=0)
        assert all(np.array_equal(x, y) for x, y in zip(a[3], b[3])), ("mc", bits, c422)
        a, b = residual_case(orc, bits, c422, seed=8), residual_case(refo, bits, c422, seed=8)
        assert all(np.array_equal(x, y) for x, y in zip(a[5], b[5])) and np.array_equal(a[6], b[6]), ("residual", bits, c422)
        if bits > 8:
            for bi in (0, 1):
                assert np.array_equal(weight_case(orc, bits, bi, 3)[3], weight_case(refo, bits, bi, 3)[3]), ("weight", bits, bi)
            assert np.array_equal(dc_case(orc, bits, c422, 4)[3], dc_case(refo, bits, c422, 4)[3]), ("dc", bits, c422)
        mb_w, mb_h = 8, 5
        rec, ext, _ = ec.deblock422_records(mb_w, mb_h, seed=9)
        ch = 16 * mb_h if c422 else 8 * mb_h
        pic = [ec.blocky((16 * mb_h, 16 * mb_w), 10, bits), ec.blocky((ch, 8 * mb_w), 11, bits), ec.blocky((ch, 8 * mb_w), 12, bits)]
        out = []
        for o in (orc, refo):
            p = [x.copy() for x in pic]
            if c422:
                hh.oracle_deblock422(o, bits, rec, ext, mb_w, mb_h, *p)
            else:
                hh.oracle_deblock(o, bits, rec, mb_w, mb_h, *p)
            out.append(p)
        assert all(np.array_equal(x, y) for x, y in zip(*out)), ("deblock", bits, c422)
