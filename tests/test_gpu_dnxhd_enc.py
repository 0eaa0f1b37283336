"""The VC-3 / DNxHD encoder on the GPU (libav_b200/csrc/dnxhd_enc.cu) against the reference encoder (oracle/_ref/libdnxhdencref.so, built on
the CPU side and carried with the tree): the CPU suite's groups byte for byte with out_info and the state after every sequence, 16 frames of
mixed CIDs across several states in one call, a capacity one byte short, a workspace one byte short, and every refusal.  Every check also
holds that nothing is written past frame_size."""
import numpy as np
import pytest

import prores_util as PU
import dnxhd_enc_util as E
from test_dnxhd_enc_cpu import GROUPS, check_refusals, sequence_cases

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="session")
def eref(built):
    lib = E.ref()
    if lib is None:
        pytest.skip("oracle/_ref not built")
    return lib


@pytest.mark.parametrize("group", sorted(GROUPS))
def test_packets_match_reference_encoder(gpu, eref, group):
    E.check(gpu.lib, eref, PU.DevMem(), GROUPS[group]())


@pytest.mark.parametrize("k", range(len(sequence_cases())))
def test_state_after_every_frame(gpu, eref, k):
    E.check_states(gpu.lib, eref, PU.DevMem(), sequence_cases()[k])


def test_mixed_cids_several_states_one_call(gpu, eref):
    """16 frames: four sequences of mixed CIDs and rate controls, each through its own state, interleaved in one call"""
    cases = [E.Case(1238, ["natural", "noise", "natural", "flat"], seed=500), E.Case(1235, ["natural", "gradient", "noise"], seed=501),
             E.Case(1243, ["natural", "natural", "noise"], interlaced=2, qmax=12, seed=502),
             E.Case(1252, ["noise", "checker", "natural"], mb_decision=E.RD, qmax=6, seed=503),
             E.Case(1260, ["natural", "flat", "noise"], mb_decision=E.RD, qmax=8, seed=504)]
    assert sum(len(c.frames) for c in cases) == 16
    E.check(gpu.lib, eref, PU.DevMem(), cases)


def test_capacity_one_byte_short(gpu, eref):
    rc, *_ = E.run(gpu.lib, eref, PU.DevMem(), [E.Case(1251, ["natural"], seed=510)], cap_delta=-1)
    assert rc == -1 and gpu.lib.avb200_last_error()
    gpu.lib.avb200_clear_error()


def test_workspace_one_byte_short(gpu, eref):
    rc, *_ = E.run(gpu.lib, eref, PU.DevMem(), [E.Case(1251, ["natural"], seed=511)], ws_delta=-1)
    assert rc == -1 and gpu.lib.avb200_last_error()
    gpu.lib.avb200_clear_error()


def test_refusals(gpu, eref):
    check_refusals(gpu.lib, eref, PU.DevMem())
