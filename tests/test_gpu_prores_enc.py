"""The ProRes encoder on the GPU (libav_b200/csrc/prores_enc.cu) against the reference encoder (oracle/_ref/libproresencref.so, built on the
CPU side and carried with the tree): the CPU suite's cases byte for byte with every slice's quantiser, 1920x1080 and 4096x2160 frames,
frames of different settings in one call, padded linesizes, a created stream, a capacity one byte short and every refusal."""
import numpy as np
import pytest

import prores_util as PU
import prores_enc_util as E
from test_prores_enc_cpu import GROUPS, check_refusals

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="session")
def eref(built):
    lib = E.ref()
    if lib is None:
        pytest.skip("oracle/_ref not built")
    return lib


def encode_and_compare(gpu, eref, cases, stream=None):
    rc, pkts, _, raws = E.run(gpu.lib, PU.DevMem(), cases, stream=stream)
    assert rc == 0, gpu.lib.avb200_last_error()
    for c, got, raw in zip(cases, pkts, raws):
        want, wq = E.ref_encode(eref, c)
        E.compare(c, got, want, wq)
        assert (raw[len(want):] == 0xCD).all(), (c, "wrote past the packet")


@pytest.mark.parametrize("group", sorted(GROUPS))
def test_packets_match_reference_encoder(gpu, eref, group):
    encode_and_compare(gpu, eref, GROUPS[group]())


@pytest.mark.parametrize("spec", [(E.FMT_422, 1920, 1080, 0, 3), (E.FMT_422, 1920, 1080, 1, 0), (E.FMT_4444, 1920, 1080, 2, 4),
                                  (E.FMT_422, 4096, 2160, 0, 3), (E.FMT_4444, 4096, 2160, 0, 4)], ids=str)
def test_large_frames(gpu, eref, spec):
    fmt, w, h, il, prof = spec
    encode_and_compare(gpu, eref, [E.Case(fmt, w, h, il, prof, 8, seed=700 + w + il)])


def test_several_settings_one_call(gpu, eref):
    """more frames than one launch takes, each with other settings: formats, field orders, profiles, slice widths, options"""
    cases = [c for k, c in enumerate(E.all_cases()) if k % 5 == 0][:19]
    encode_and_compare(gpu, eref, cases)


def test_padded_linesizes(gpu, eref):
    cases = [E.Case(E.FMT_422, 200, 72, 1, 3, 4, pad=6, seed=710), E.Case(E.FMT_4444, 120, 40, 0, 4, 2, pad=130, seed=711),
             E.Case(E.FMT_444, 72, 35, 2, 2, 8, pad=2, seed=712)]
    encode_and_compare(gpu, eref, cases)


def test_created_stream(gpu, eref):
    s = gpu.lib.avb200_stream_create()
    assert s
    try:
        encode_and_compare(gpu, eref, [E.Case(E.FMT_4444, 160, 96, 1, 4, 4, seed=720), E.Case(E.FMT_422, 96, 48, 0, 0, 8, bits_per_mb=128,
                                                                                         content="noise", seed=721)], stream=s)
    finally:
        gpu.lib.avb200_stream_destroy(s)


def test_capacity_one_byte_short(gpu, eref):
    cases = [E.Case(E.FMT_422, 1920, 64, 0, 3, 8, seed=730), E.Case(E.FMT_4444, 56, 34, 2, 4, 4, seed=731)]
    want = [E.ref_encode(eref, c)[0] for c in cases]
    rc, _, sizes, raws = E.run(gpu.lib, PU.DevMem(), cases, cap_delta=[(len(w), -1) for w in want])
    assert rc == 0
    for w, s, raw in zip(want, sizes, raws):
        assert s == -len(w) and (raw == 0xCD).all()
    rc, pkts, _, raws = E.run(gpu.lib, PU.DevMem(), cases, cap_delta=[(len(w), 0) for w in want])
    assert rc == 0
    for w, p, raw in zip(want, pkts, raws):
        assert np.array_equal(p, w) and (raw[len(w):] == 0xCD).all()


def test_refusals(gpu):
    assert len(check_refusals(gpu.lib, PU.DevMem())) == 38
    gpu.lib.avb200_clear_error()
