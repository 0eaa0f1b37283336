"""The arithmetic of the batched H.264 inter prediction (libav_b200/csrc/h264_mc_block.cuh: one thread per 4x4 block, packed-byte dot
products) compiled for the host and run block after block over synthetic record lists -- every quarter-sample position, every partition
size, vectors that leave the picture, `avg` second directions, stacked pictures, unaligned reference planes -- against the compiled
reference's qpel / chroma tables (tests/h264_util.py::oracle_mc).  TEST INFRASTRUCTURE: the GPU runs the same function per lane
(tests/test_gpu_h264.py, tests/test_gpu_h264chain.py)."""
import numpy as np
import pytest

from libav_b200 import synth
import h264_util as hu
import hostsim_build


@pytest.fixture
def mcsim(built):
    return hostsim_build.fresh()


def run_sim(lib, rec, refs, y, cb, cr, pw, ph, votes):
    planes = np.array([[p.ctypes.data for p in r] for r in refs], np.uint64)
    assert lib.hostsim_h264_mc(rec.ctypes.data, rec.shape[0], planes.ctypes.data, y.ctypes.data, cb.ctypes.data, cr.ctypes.data,
                               y.strides[0], cb.strides[0], pw, ph, votes) == 0


@pytest.mark.parametrize("mb_w,mb_h,max_mv", [(6, 4, 40), (11, 7, 130), (3, 2, 300)])
def test_every_position_and_partition(mcsim, refo, mb_w, mb_h, max_mv):
    refs = [synth.h264_picture(mb_w, mb_h, seed=11), synth.h264_picture(mb_w, mb_h, seed=12)]
    rec = synth.h264_mc_work(mb_w, mb_h, seed=mb_w, max_mv=max_mv)
    fr = {(int(r["mvx"] + 4 * r["x"]) & 3, int(r["mvy"] + 4 * r["y"]) & 3) for r in rec}
    assert len(fr) >= (16 if mb_w > 6 else 12)                   # (all) sixteen quarter-sample positions occur
    want = [np.zeros((16 * mb_h, 16 * mb_w), np.uint8), np.zeros((8 * mb_h, 8 * mb_w), np.uint8), np.zeros((8 * mb_h, 8 * mb_w), np.uint8)]
    hu.oracle_mc(refo, rec, refs, *want, pad=96)
    for votes in (0, 1):
        got = [np.full_like(w, 0x5A) for w in want]
        run_sim(mcsim, rec, refs, *got, 16 * mb_w, 16 * mb_h, votes)
        for g, w, name in zip(got, want, "y cb cr".split()):
            assert np.array_equal(g, w), (votes, name, np.argwhere(g != w)[:5].tolist())


def test_stacked_pictures_and_unaligned_references(mcsim, refo):
    """two pictures stacked vertically (a block of picture 1 must clamp inside picture 1 of its reference), and reference planes at odd
    addresses (the byte path of every fetch)"""
    mb_w, mb_h, P = 5, 3, 2
    W, H = 16 * mb_w, 16 * mb_h
    refs1 = [[synth.h264_picture(mb_w, mb_h, seed=20 + 2 * k + j) for k in range(P)] for j in range(2)]      # [ref][picture]
    recs, want = [], []
    for k in range(P):
        rec = synth.h264_mc_work(mb_w, mb_h, seed=30 + k, max_mv=90)
        w = [np.zeros((H, W), np.uint8), np.zeros((H // 2, W // 2), np.uint8), np.zeros((H // 2, W // 2), np.uint8)]
        hu.oracle_mc(refo, rec, [refs1[0][k], refs1[1][k]], *w, pad=64)
        want.append(w)
        rec = rec.copy(); rec["y"] = rec["y"] + k * H; recs.append(rec)
    rec = np.concatenate(recs)
    stacked = [[np.concatenate([refs1[j][k][p] for k in range(P)]) for p in range(3)] for j in range(2)]
    for shift in (0, 1):
        if shift:                                                # the same bytes one byte further: nothing is 4-byte aligned any more
            hold = [[np.zeros(p.size + 8, np.uint8) for p in r] for r in stacked]
            use = [[h[1:1 + p.size].reshape(p.shape) for h, p in zip(hr, r)] for hr, r in zip(hold, stacked)]
            for ur, r in zip(use, stacked):
                for u, p in zip(ur, r):
                    u[...] = p
        else:
            use = stacked
        got = [np.zeros((P * H, W), np.uint8), np.zeros((P * H // 2, W // 2), np.uint8), np.zeros((P * H // 2, W // 2), np.uint8)]
        run_sim(mcsim, rec, use, *got, W, H, 1)
        for p in range(3):
            assert np.array_equal(got[p], np.concatenate([want[k][p] for k in range(P)])), (shift, p)


@pytest.mark.parametrize("modes,shift", [((0, 1), 0), ((0,), 0), ((1,), 0), ((0, 1, 3), 0), ((0, 1), 1)])
def test_residual_kernel_on_the_host(mcsim, refo, modes, shift):
    """libav_b200/csrc/h264_residual.cu (one lane per 4x4 / 8x8 block, transforms in registers) compiled for the host: pixels AND the
    consumed coefficient arena against the reference's h264_idct_add16 / add16intra / idct_add8; shift = 1 puts the macroblocks at odd
    byte offsets (the byte path of the pixel rows).  Transform-8x8 macroblocks exchange rows and columns between lanes through shared
    memory: that path is GPU-only (tests/test_gpu_h264.py::test_residual_batch, tests/test_gpu_h264chain.py)"""
    mb_w, mb_h = 9, 6
    rec, coeffs, nnzc = synth.h264_residual_work(mb_w, mb_h, seed=3 + len(modes), modes=modes)
    y, cb, cr = synth.h264_picture(mb_w, mb_h + 1, seed=4)            # one spare macroblock row: the shifted offsets stay inside
    if shift:
        rec = rec.copy(); rec["luma_off"] += 1; rec["chroma_off"] += 1
    wy, wcb, wcr, wco = y.copy(), cb.copy(), cr.copy(), coeffs.copy()
    hu.oracle_residual(refo, rec, wco, nnzc, wy, wcb, wcr)
    gy, gcb, gcr, gco = y.copy(), cb.copy(), cr.copy(), np.ascontiguousarray(coeffs.copy())
    assert mcsim.hostsim_h264_residual(rec.ctypes.data, rec.shape[0], gco.ctypes.data, 768, nnzc.ctypes.data, gy.ctypes.data, gcb.ctypes.data, gcr.ctypes.data,
                                       gy.strides[0], gcb.strides[0]) == 0
    assert np.array_equal(gy, wy) and np.array_equal(gcb, wcb) and np.array_equal(gcr, wcr)
    assert np.array_equal(gco, wco), "consumed coefficients"
    assert not np.array_equal(gy, y)
