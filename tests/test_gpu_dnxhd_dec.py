"""The VC-3 / DNxHD decoder on the GPU (libav_b200/csrc/dnxhd_dec.cu) against the reference decoder (oracle/_ref/libdnxhddecref.so, built on
the CPU side and carried with the tree), one fresh context per packet, every plane byte for byte with the sentinel: the CPU suite's real
and synthesised packets, batches of 1, 16 and 64 1080p frames in one call, 4:4:4 10-bit frames, gray, padded linesizes, mixed CIDs, and
every refusal."""
import pytest

import prores_util as PU
import dnxhd_dec_util as D
import dnxhd_enc_util as E
from test_dnxhd_dec_cpu import REAL, SYNTH, check_refusals, synth

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="session")
def dref(built):
    lib = D.ref()
    if lib is None or E.ref() is None:
        pytest.skip("oracle/_ref not built")
    return lib


@pytest.fixture(scope="session")
def eref(dref):
    return E.ref()


@pytest.mark.parametrize("name", sorted(REAL))
def test_real_packets(gpu, dref, eref, name):
    cid, contents, il, mbd = REAL[name]
    D.check(gpu.lib, dref, PU.DevMem(), D.real_packets(eref, cid, contents, interlaced=il, mb_decision=mbd, seed=7 + len(name)))


@pytest.mark.parametrize("name", sorted(SYNTH))
def test_synthesised_packets(gpu, dref, name):
    D.check(gpu.lib, dref, PU.DevMem(), [synth(dref, name)])


@pytest.mark.parametrize("n", [1, 16, 64])
def test_1080p_batches(gpu, dref, eref, n):
    """n 1080p packets in one call: 8-bit, 10-bit and interlaced CIDs in turn"""
    cids = (1238, 1235, 1243, 1253)
    pool = {c: D.real_packets(eref, c, ["natural", "noise"], seed=40 + c) for c in cids}
    pk = [pool[cids[k % 4]][(k // 4) % 2] for k in range(n)]
    D.check(gpu.lib, dref, PU.DevMem(), pk)


def test_444_10bit_frames(gpu, dref):
    pk = [D.synth(dref, D.Synth(1256, seed=60 + k, is444=True, eob=0.3)) for k in range(2)]
    D.check(gpu.lib, dref, PU.DevMem(), pk)


def test_gray_padded_mixed(gpu, dref, eref):
    pk = D.real_packets(eref, 1251, ["natural"], seed=3)
    D.check(gpu.lib, dref, PU.DevMem(), pk, gray=1)
    D.check(gpu.lib, dref, PU.DevMem(), pk + [synth(dref, n) for n in ("444", "mbaff_1260", "sar", "fields_bff")], pad=40)


def test_refusals(gpu, dref, eref):
    check_refusals(gpu.lib, dref, eref, PU.DevMem())
