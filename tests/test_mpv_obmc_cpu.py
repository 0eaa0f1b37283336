"""CPU: H.263 overlapped block motion compensation in ff_mpv_motion_batch_cuda.  The product (libav_b200/csrc/mpv_obmc.cuh through
mpv_mc.cu, compiled for the host by tests/hostsim/mpv_mc_hostsim.cpp) and the plain-C port (oracle/port/orc_mpvobmc.c) against the
reference's real ff_mpv_motion with s->obmc set (oracle/_ref/libmpvobmcref.so), whose tables hold each record's raw entries when it runs:
no_rounding 0 and 1; 16X16 and 8X8 records; intra and missing neighbours on every side; vectors far outside, at and next to every edge,
custom sizes; right neighbours whose entries disagree with that macroblock's own vectors (the decoder's stale tables); B pictures, where
obmc is ignored; a 16X16 macroblock's chroma through chroma_4mv_motion, which differs from the 16X16 chroma path; the refusals."""
import ctypes as C

import numpy as np
import pytest

import hostsim_build
import mpv_mc_cases as M
import mpv_obmc_cases as O


@pytest.fixture(scope="module")
def obref(built):
    lib = O.ref_lib()
    if lib is None:
        pytest.skip("oracle/_ref not built (no reference tree in this environment)")
    return lib


@pytest.fixture
def obsim(built):
    return hostsim_build.fresh()


@pytest.fixture(scope="module")
def obport(built):
    return O.port_lib()


CASES = [(no_rnd, ragged, stale) for no_rnd in (0, 1) for ragged in (0, 1, 2) for stale in (0.0, 0.5)]


@pytest.mark.parametrize("no_rnd,ragged,stale", CASES)
def test_hostsim_matches_reference(obref, obsim, no_rnd, ragged, stale):
    for seed in range(3):
        pic = O.obmc_picture(np.random.default_rng(100 * seed + 10 * no_rnd + ragged), 6, 5, no_rnd=no_rnd, ragged=ragged, stale=stale)
        got, rej = O.run_sim(obsim, [pic])
        assert rej == 0
        d = M.first_diff(got[0], O.run_ref(obref, pic))
        assert d is None, (seed, d)


@pytest.mark.parametrize("no_rnd,ragged,stale", CASES)
def test_port_matches_reference(obref, obport, no_rnd, ragged, stale):
    for seed in range(3):
        pic = O.obmc_picture(np.random.default_rng(700 + 100 * seed + 10 * no_rnd + ragged), 6, 5, no_rnd=no_rnd, ragged=ragged, stale=stale)
        d = M.first_diff(O.run_ref(obport, pic), O.run_ref(obref, pic))
        assert d is None, (seed, d)


def test_edges_intra_and_tiny_pictures(obref, obsim, obport):
    """every macroblock at an edge, most vectors at / next to / far outside one, neighbours intra half of the time; 1 x 1 .. 3 x 2 pictures"""
    for seed in range(30):
        rng = np.random.default_rng(seed)
        w, h = int(rng.integers(1, 4)), int(rng.integers(1, 3))
        pic = O.obmc_picture(rng, w, h, no_rnd=seed & 1, ragged=seed % 3, intra=0.5, stale=0.5, far=0.3, edge=0.6)
        want = O.run_ref(obref, pic)
        got, rej = O.run_sim(obsim, [pic])
        assert rej == 0 and M.first_diff(got[0], want) is None, (seed, M.first_diff(got[0], want))
        assert M.first_diff(O.run_ref(obport, pic), want) is None, seed


def test_stale_right_neighbour_is_what_counts(obref, obsim):
    """the same picture with the right neighbours' entries replaced: the result follows the record, not the neighbour's own vectors"""
    rng = np.random.default_rng(5)
    pic = O.obmc_picture(rng, 5, 4, stale=0.0, intra=0.0)
    base = O.run_ref(obref, pic)
    pic.obmc["right"] += np.int16(6)
    want = O.run_ref(obref, pic)
    assert M.first_diff(want, base) is not None
    got, _ = O.run_sim(obsim, [pic])
    assert M.first_diff(got[0], want) is None


def test_16x16_chroma_goes_through_chroma_4mv(obref, obsim):
    """16X16 macroblocks whose neighbours share their vector: the chroma comes from chroma_4mv_motion of four times the vector, which clips
    its position to [-8, width / 2] and drops the half-sample bit there where the 16X16 path reads on to h_edge_pos: in an H.263
    custom-size picture with vectors at the right / bottom edges the two give different chroma"""
    rng = np.random.default_rng(8)
    pic = O.obmc_picture(rng, 5, 4, ragged=2, intra=0.0, stale=0.0, far=0.0, edge=0.9)
    pic.recs["mv_type"] = M.T16X16
    for r, o in zip(pic.recs, pic.obmc):
        o["mv"][:] = r["mv"][0, 0]
        o["top"][:] = o["left"][:] = o["right"][:] = r["mv"][0, 0]
    want = O.run_ref(obref, pic)
    plain = M.run_ref(M.ref_lib(), pic)
    assert not np.array_equal(want[1], plain[1]) and not np.array_equal(want[2], plain[2])
    got, _ = O.run_sim(obsim, [pic])
    assert M.first_diff(got[0], want) is None


def test_b_pictures_ignore_obmc(obref, obsim):
    pic = O.obmc_picture(np.random.default_rng(9), 6, 4, b=1)
    want = M.run_ref(M.ref_lib(), pic)
    assert M.first_diff(O.run_ref(obref, pic), want) is None
    got, rej = O.run_sim(obsim, [pic])
    assert rej == 0 and M.first_diff(got[0], want) is None


def test_mixed_call_and_backward_records(obref, obsim):
    """plain and OBMC pictures in one call, more than one launch each; OBMC records with a backward direction are counted, not run"""
    pics = [O.obmc_picture(np.random.default_rng(20 + i), 3, 3, no_rnd=i & 1) for i in range(18)]
    plain = []
    for i in range(3):
        p = O.obmc_picture(np.random.default_rng(60 + i), 3, 3)
        plain.append(p)
    pics[3].recs["mv_dir"][:2] = [2, 3]
    frames = [[a.copy() for a in p.frame] for p in pics + plain]
    recs = [np.ascontiguousarray(p.recs) for p in pics + plain]
    obs = [np.ascontiguousarray(p.obmc) for p in pics + plain]
    arr = O.structs(pics + plain, [[a.ctypes.data for a in f] for f in frames], [r.ctypes.data for r in recs], [o.ctypes.data for o in obs],
                    [[a.ctypes.data for a in p.last] for p in pics + plain], [[a.ctypes.data for a in p.next] for p in pics + plain])
    for k in range(len(pics), len(pics) + len(plain)):
        arr[k].obmc, arr[k].obmc_recs = 0, None
    rej = np.zeros(1, np.uint32)
    assert obsim.ff_mpv_motion_batch_cuda(C.cast(arr, C.c_void_p), len(arr), rej.ctypes.data, None) == 0
    assert rej[0] == 2
    for i, p in enumerate(pics):
        assert M.first_diff(frames[i], O.run_ref(obref, p)) is None, i
    for k, p in enumerate(plain):
        assert M.first_diff(frames[len(pics) + k], M.run_ref(M.ref_lib(), p)) is None, k


@pytest.mark.parametrize("field,value", [("quarter_sample", 1), ("out_format", 0), ("obmc_recs", None)])
def test_refusals_change_nothing(obsim, field, value):
    pic = O.obmc_picture(np.random.default_rng(3), 4, 3)
    frame = [a.copy() for a in pic.frame]
    recs, ob = np.ascontiguousarray(pic.recs), np.ascontiguousarray(pic.obmc)
    arr = O.structs([pic], [[a.ctypes.data for a in frame]], [recs.ctypes.data], [ob.ctypes.data], [[a.ctypes.data for a in pic.last]],
                    [[a.ctypes.data for a in pic.next]])
    setattr(arr[0], field, value)
    rej = np.zeros(1, np.uint32)
    obsim.avb200_clear_error()
    assert obsim.ff_mpv_motion_batch_cuda(C.cast(arr, C.c_void_p), 1, rej.ctypes.data, None) == -1
    assert b"OBMC" in obsim.avb200_last_error()
    assert all(np.array_equal(a, b) for a, b in zip(frame, pic.frame)) and rej[0] == 0
