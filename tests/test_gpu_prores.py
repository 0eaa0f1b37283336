"""ProRes reconstruction on the GPU (libav_b200/csrc/prores.cu) against the reference (oracle/_ref/libproresref.so, built on the CPU side
and carried with the tree): the ProresDSPContext slot checkasm-style, the batch call under each kernel its dispatcher picks, the picture call
on reference-encoded streams (every chroma format, field order and profile, alpha, right-edge slices, 1080-line frames, several pictures
in one call) and every refusal."""
import ctypes as C

import numpy as np
import pytest

import prores_util as U
from libav_b200 import tables
from test_prores_cpu import check_refusals

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="session")
def pref(built):
    lib = U.ref()
    if lib is None:
        pytest.skip("oracle/_ref not built")
    return lib


def test_slot_checkasm(gpu, pref):
    """the slot against prores_idct_put_c on the edge blocks, with the destination inside a canvas whose border must stay untouched"""
    t = tables.ProresDSPContext()
    gpu.lib.ff_proresdsp_init_cuda(C.byref(t))
    assert t.idct_permutation_type == 0 and list(t.idct_permutation) == list(range(64))
    blocks, qm, _ = U.edge_blocks(3)
    for k in range(0, len(blocks), 5):
        ls = (24, 34, 48)[k % 3]
        canvas = np.random.default_rng(k).integers(0, 65536, (12, ls // 2), dtype=np.uint16)
        want = canvas.copy()
        wb = blocks[k].copy(); gb = blocks[k].copy()
        pref.ref_prores_idct_put(U.P(want, 2 * ls + 4), ls, U.P(wb), U.P(qm[k]))
        t.idct_put(C.cast(canvas.ctypes.data + 2 * ls + 4, C.POINTER(C.c_uint16)), ls,
                   gb.ctypes.data_as(C.POINTER(C.c_int16)), qm[k].ctypes.data_as(C.POINTER(C.c_int16)))
        assert np.array_equal(canvas, want) and np.array_equal(gb, wb), k
    gpu.check(0, "slot")


@pytest.mark.parametrize("layout", ["staged", "staged_no_qidx", "odd_pitch", "misaligned_blocks", "misaligned_qmats", "staged_unaligned_frame"])
def test_batch_every_kernel(gpu, pref, layout):
    """staged kernel (16-byte aligned blocks and matrices, pitch a multiple of 16) and the thread-per-block kernel for the rest"""
    blocks, qm, qidx = U.edge_blocks(4)
    blocks = np.concatenate([blocks] * 3)                        # several groups per warp, a ragged last group
    qidx = np.concatenate([qidx] * 3)
    if layout == "staged_no_qidx":
        qm, qidx = qm[5:6], np.zeros(len(blocks), np.uint32)
    want_b, want_s = U.ref_idct_put(pref, blocks, qm, qidx)
    kw = {"odd_pitch": dict(pitch_extra=2), "misaligned_blocks": dict(block_pad=2), "misaligned_qmats": dict(qmat_pad=8),
          "staged_unaligned_frame": dict(frame_pad=2)}.get(layout, {})
    rc, got_b, got_s = U.run_batch(gpu.lib, U.DevMem(), blocks, qm, None if layout == "staged_no_qidx" else qidx, **kw)
    assert rc == 0, gpu.last_error()
    assert np.array_equal(got_b, want_b), np.flatnonzero((got_b != want_b).any(1))[:8]
    assert np.array_equal(got_s, want_s), np.flatnonzero((got_s != want_s).reshape(len(blocks), -1).any(1))[:8]


def test_batch_large(gpu, pref):
    """2^18 blocks through the staged kernel (the grid-stride loop and the double buffer): checked against the reference on a sample"""
    r = np.random.default_rng(9)
    n = 1 << 18
    blocks = (r.integers(-400, 400, (n, 64)) * (r.random((n, 64)) < 0.15)).astype(np.int16)
    qm = r.integers(1, 64 * 8, (16, 64)).astype(np.int16)
    qidx = r.integers(0, 16, n).astype(np.uint32)
    rc, got_b, got_s = U.run_batch(gpu.lib, U.DevMem(), blocks, qm, qidx, tiles_per_row=512)
    assert rc == 0
    pick = r.choice(n, 4096, replace=False)
    want_b, want_s = U.ref_idct_put(pref, blocks[pick], qm, qidx[pick])
    assert np.array_equal(got_b[pick], want_b) and np.array_equal(got_s[pick], want_s)


@pytest.mark.parametrize("spec", U.STREAMS, ids=str)
def test_pictures_match_reference_decoder(gpu, pref, spec):
    d = U.Decoded(pref, spec)
    rc, got = U.run_pictures(gpu.lib, U.DevMem(), [d])
    assert rc == 0, gpu.last_error()
    U.check_frame(d, got[0])


def test_pictures_unaligned_coefficients(gpu, pref):
    """coefficient buffers off 16-byte alignment take the thread-per-block kernel"""
    decs = [U.Decoded(pref, spec, seed=40 + k) for k, spec in enumerate(U.SMALL_STREAMS[:5])]
    rc, got = U.run_pictures(gpu.lib, U.DevMem(), decs, block_pad=2)
    assert rc == 0
    for d, g in zip(decs, got):
        U.check_frame(d, g)


def test_pictures_scrambled_quantisers(gpu, pref):
    decs = [U.Decoded(pref, spec, seed=11 + k, scrambled=True) for k, spec in enumerate(U.SMALL_STREAMS)]
    rc, got = U.run_pictures(gpu.lib, U.DevMem(), decs)
    assert rc == 0
    for d, g in zip(decs, got):
        U.check_frame(d, g)


def test_pictures_mixed_geometry_one_call(gpu, pref):
    """more pictures than one launch takes, of different geometry, in one call"""
    specs = U.SMALL_STREAMS + [U.STREAMS[-3]]
    decs = [U.Decoded(pref, spec, seed=20 + k) for k, spec in enumerate(specs)]
    assert sum(d.rec.n_pics for d in decs) > 8
    rc, got = U.run_pictures(gpu.lib, U.DevMem(), decs)
    assert rc == 0
    for d, g in zip(decs, got):
        U.check_frame(d, g)


def test_refusals(gpu, pref):
    d = U.Decoded(pref, U.SMALL_STREAMS[0])
    assert len(check_refusals(gpu.lib, U.DevMem(), d)) == 19
    gpu.check(0, "after refusals")
