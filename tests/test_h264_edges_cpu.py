"""The edge cases of tests/h264_edge_cases.py on the CPU: the batched H.264 inter prediction (h264_mc_block.cuh) and the register-resident
residual kernel (h264_residual.cu, 4x4 paths) compiled for the host and run against the compiled reference (`refo`) -- far vectors,
every partition shape, decoder-layout pictures inside poisoned allocations, odd picture sizes, any record order, int16 wrap-around
and the dispatch rules of the residual add.  The plain-C port is pinned to the reference on the same cases, so it stays a faithful
checker where the reference is not built.  The GPU runs the same cases through every kernel choice (tests/test_gpu_h264_edges.py)."""
import numpy as np
import pytest

from libav_b200 import synth
import h264_edge_cases as ec
import h264_util as hu
import hostsim_build

MB_W, MB_H = 12, 8
TIGHT = ec.Layout("tight", 0, 0)
MC_LAYOUTS = [TIGHT, ec.PAD4, ec.PAD2, ec.SHIFT1, ec.SHIFT2, ec.ODD_UV, ec.ODD_CB, ec.REF1]


@pytest.fixture(scope="module")
def sim(built):
    return hostsim_build.fresh()


@pytest.fixture(scope="module")
def mc_case(refo):
    refs = [synth.h264_picture(MB_W, MB_H, seed=71), synth.h264_picture(MB_W, MB_H, seed=72)]
    dst = synth.h264_picture(MB_W, MB_H, seed=73)
    rec = ec.mc_records(MB_W, MB_H, seed=74)
    return refs, dst, rec, ec.oracle_mc(refo, rec, refs, dst)


def sim_mc(lib, rec, refs, dst, lay, pw, ph, votes):
    """hostsim_h264_mc with every plane placed by `lay`; checks the poisoned bytes and returns the pictures"""
    d = [lay.place(p, chroma=i > 0) for i, p in enumerate(dst)]
    r = [[lay.place(p, chroma=i > 0, ref=True) for i, p in enumerate(rp)] for rp in refs]
    planes = np.array([[v.ctypes.data for _, v in rp] for rp in r], np.uint64)
    assert lib.hostsim_h264_mc(rec.ctypes.data, rec.shape[0], planes.ctypes.data, d[0][1].ctypes.data, d[1][1].ctypes.data,
                               d[2][1].ctypes.data, d[0][1].strides[0], d[1][1].strides[0], pw, ph, votes) == 0
    for (b, v), p in zip([x for rp in r for x in rp], [p for rp in refs for p in rp]):
        ec.Layout.check(b, v, p, "reference")
    return d


@pytest.mark.parametrize("lay", MC_LAYOUTS, ids=repr)
def test_mc_far_vectors_in_decoder_layout(sim, mc_case, lay):
    refs, dst, rec, want = mc_case
    for votes in (0, 1):
        got = sim_mc(sim, rec, refs, dst, lay, 16 * MB_W, 16 * MB_H, votes)
        for (b, v), w, name in zip(got, want, ("y", "cb", "cr")):
            ec.Layout.check(b, v, w, (votes, name))


@pytest.mark.parametrize("pw,ph", [(16 * MB_W - 1, 16 * MB_H), (16 * MB_W, 16 * MB_H - 1), (16 * MB_W - 3, 16 * MB_H - 3)])
def test_mc_odd_picture_size(sim, refo, mc_case, pw, ph):
    """clamping at an odd width / height: the reference planes end at pw x ph, the partitions still cover whole macroblocks (ph stays
    above the last partition row: a record at y >= pic_h belongs to the next stacked picture)"""
    refs, dst, rec, _ = mc_case
    want = ec.oracle_mc(refo, rec, refs, dst, pw, ph)
    got = sim_mc(sim, rec, refs, dst, ec.PAD4, pw, ph, 1)
    for (b, v), w in zip(got, want):
        ec.Layout.check(b, v, w)


def test_mc_any_record_order_and_batch_size(sim, refo, mc_case):
    refs, dst, rec, want = mc_case
    perm = rec[np.random.default_rng(5).permutation(rec.shape[0])]
    assert any(perm["avg"][k] and not perm["avg"][k + 1] for k in range(perm.shape[0] - 1))        # avg records ahead of put records
    got = sim_mc(sim, perm, refs, dst, ec.PAD4, 16 * MB_W, 16 * MB_H, 1)
    for (b, v), w in zip(got, want):
        ec.Layout.check(b, v, w, "permuted")
    for n in (1, 31, 33, 129):
        sub = rec[np.sort(np.random.default_rng(n).choice(rec.shape[0], n, replace=False))]
        w = ec.oracle_mc(refo, sub, refs, dst)
        got = sim_mc(sim, sub, refs, dst, ec.PAD4, 16 * MB_W, 16 * MB_H, 1)
        for (b, v), wp in zip(got, w):
            ec.Layout.check(b, v, wp, n)


@pytest.mark.parametrize("lay,stride", [(TIGHT, 768), (ec.PAD4, 768), (ec.PAD4, 776)], ids=["tight", "pad4", "pad4-776"])
def test_residual_wraparound_and_dispatch(sim, refo, lay, stride):
    """pixels, the consumed arena and the untouched bytes around both; transform-8x8 macroblocks exchange data between lanes and run on
    the GPU only (tests/test_gpu_h264_edges.py)"""
    mb_w, mb_h = 9, 6
    rec, coeffs, nnzc = ec.residual_records(mb_w, mb_h, seed=21, modes=(0, 1, 3))
    pic = synth.h264_picture(mb_w, mb_h, seed=22)
    want = [p.copy() for p in pic]
    want_co = coeffs.copy()
    hu.oracle_residual(refo, rec, want_co, nnzc, *want)
    d = [lay.place(p, chroma=i > 0) for i, p in enumerate(pic)]
    ls, uvls = d[0][1].strides[0], d[1][1].strides[0]
    r2 = ec.relayout_residual(rec, 16 * mb_w, ls, uvls)
    arena = np.full((coeffs.shape[0], stride), 0x5A5A, np.int16)
    arena[:, :768] = coeffs
    assert sim.hostsim_h264_residual(r2.ctypes.data, r2.shape[0], arena.ctypes.data, stride, nnzc.ctypes.data, d[0][1].ctypes.data,
                                     d[1][1].ctypes.data, d[2][1].ctypes.data, ls, uvls) == 0
    for (b, v), w in zip(d, want):
        ec.Layout.check(b, v, w)
    assert np.array_equal(arena[:, :768], want_co), np.argwhere(arena[:, :768] != want_co)[:5].tolist()
    assert (arena[:, 768:] == 0x5A5A).all()
    assert (want_co != 0).any()                                       # blocks the dispatchers skip, and AC left behind, stay


def test_port_pinned_to_reference_residual(orc, refo):
    """the port as a checker of the wrap-around and dispatch-rule cases, 4x4 and 8x8"""
    rec, coeffs, nnzc = ec.residual_records(8, 6, seed=31)
    pic = synth.h264_picture(8, 6, seed=32)
    out = []
    for o in (orc, refo):
        p, co = [x.copy() for x in pic], coeffs.copy()
        hu.oracle_residual(o, rec, co, nnzc, *p)
        out.append((p, co))
    for a, b in zip(out[0][0], out[1][0]):
        assert np.array_equal(a, b)
    assert np.array_equal(out[0][1], out[1][1])


def test_port_pinned_to_reference_mc(orc, refo, mc_case):
    refs, dst, rec, want = mc_case
    for a, b in zip(ec.oracle_mc(orc, rec, refs, dst), want):
        assert np.array_equal(a, b)


@pytest.mark.parametrize("bi", [0, 1])
def test_port_pinned_to_reference_weight(orc, refo, bi):
    rec, plane, src = ec.weight_records(bi, seed=41)
    out = []
    for o in (orc, refo):
        p = plane.copy()
        hu.oracle_weight(o, rec, p, src if bi else None)
        out.append(p)
    assert np.array_equal(out[0], out[1])


def test_port_pinned_to_reference_deblock(orc, refo):
    mb_w, mb_h = 9, 6
    rec = ec.deblock_records(mb_w, mb_h, seed=51)
    pic = [ec.blocky((16 * mb_h, 16 * mb_w), 52), ec.blocky((8 * mb_h, 8 * mb_w), 53), ec.blocky((8 * mb_h, 8 * mb_w), 54)]
    out = []
    for o in (orc, refo):
        p = [x.copy() for x in pic]
        hu.oracle_deblock(o, rec, mb_w, mb_h, *p)
        out.append(p)
    for a, b in zip(*out):
        assert np.array_equal(a, b)
    assert (np.abs(out[1][0].astype(int) - pic[0]) > 12).sum() > 50           # the large-tc and strong filters did act
