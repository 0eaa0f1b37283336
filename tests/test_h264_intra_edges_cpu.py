"""The intra edge cases of tests/h264_intra_cases.py on the CPU: the generator produces every case it exists for, its availability masks
are the ones synth.h264_intra_work derives where both apply, and the plain-C port is pinned to the compiled reference (`refo`) on every
picture of the matrix, int16 wrap-around included, so it stays a faithful checker where the reference is not built.  The GPU runs the
same pictures through the batch calls (tests/test_gpu_h264_intra_edges.py)."""
import collections

import numpy as np
import pytest

from libav_b200 import synth
import h264_hbd_util as hh
import h264_intra_cases as ic
import h264_util as hu


@pytest.fixture(scope="module")
def cases():
    return ic.matrix_cases()


def test_generator_covers_its_cases(cases):
    seen = collections.Counter()
    for c in cases.values():
        seen.update(c["seen"])
    ic.assert_coverage(seen)
    assert all(c["slices"] > 1 for (w, h, s, _), c in cases.items() if s and w * h > 1)


@pytest.mark.parametrize("mb_w,mb_h", ic.SIZES)
def test_masks_equal_synth_on_single_slice_pictures(cases, mb_w, mb_h):
    """one slice, constrained_intra_pred off: availability follows from the picture border alone, as in synth.h264_intra_work"""
    rec = cases[mb_w, mb_h, False, False]["rec"]
    old, _, _ = synth.h264_intra_work(mb_w, mb_h, seed=3)
    intra = rec["kind"] != 0
    assert intra.any()
    for f in ("topleft", "topright"):
        assert np.array_equal(rec[f][intra], old[f][intra]), f


def _pin(orc, refo, run, planes, co):
    out = []
    for o in (orc, refo):
        p, c = [x.copy() for x in planes], co.copy()
        run(o, c, p)
        out.append((p, c))
    for a, b in zip(out[0][0], out[1][0]):
        assert np.array_equal(a, b), np.argwhere(a != b)[:5].tolist()
    assert np.array_equal(out[0][1], out[1][1])
    assert any((a != b).any() for a, b in zip(out[1][0], planes))


@pytest.mark.parametrize("key", [(w, h, s, c) for (w, h) in ic.SIZES for (s, c) in ic.VARIANTS], ids=lambda k: "%dx%d-slices%d-cip%d" % k)
def test_port_pinned_to_reference_intra(orc, refo, cases, key):
    mb_w, mb_h = key[:2]
    c = cases[key]
    _pin(orc, refo, lambda o, co, p: hu.oracle_intra(o, c["rec"], co, c["nnzc"], mb_w, mb_h, *p), c["planes"], c["coeffs"])


@pytest.mark.parametrize("bits,c422", [(9, 0), (10, 0), (8, 1), (9, 1), (10, 1)])
def test_port_pinned_to_reference_intra_hbd_422(orc, refo, bits, c422):
    """the cases the _hbd / _422 calls run on the GPU: int32 coefficients up to +-2^20 above 8 bit, int16 wrap-around at 8 bit"""
    for (s, cip) in ic.VARIANTS:
        c = ic.intra_case(11, 7, 70 + 2 * s + cip, s, cip, bits, c422)
        _pin(orc, refo, lambda o, co, p: hh.oracle_intra(o, bits, c["rec"], co, c["nnzc"], 11, 7, *p, c422=c422), c["planes"], c["coeffs"])
