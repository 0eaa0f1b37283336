"""The ProRes decoder on the GPU (libav_b200/csrc/prores_dec.cu) against the reference decoder with the checked reader
(oracle/_ref/libproresdecref.so, built on the CPU side and carried with the tree), one fresh context per packet, every plane byte for byte
with the sentinel and the alpha plane: the CPU suite's packets and header edits (the zero_plane_dc_* edits reach decode_vlc_codeword's
shift counts past 32, where CUDA's >> differs from the reference's), packets this library's GPU encoder wrote and decoded without
leaving the device, batches of 1, 16 and 64 packets at 1920x1080 and 4096x2160 mixing formats and field orders, padded linesizes, and
every refusal."""
import ctypes as C

import numpy as np
import pytest

import prores_util as PU
import prores_enc_util as E
import prores_dec_util as D
from libav_b200 import tables
from test_prores_dec_cpu import EDITS, REAL, check_refusals, edited, real

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
def test_reference_encoder_packets(gpu, dref, eref, name):
    D.check(gpu.lib, dref, PU.DevMem(), [real(eref, name)])


@pytest.mark.parametrize("name", sorted(EDITS))
def test_header_edits(gpu, dref, eref, name):
    D.check(gpu.lib, dref, PU.DevMem(), [edited(eref, name)])


def test_gpu_encoder_packets_stay_on_device(gpu, dref):
    """this library's encoder writes the packets; the decoder reads them where the encoder left them"""
    cases = [E.Case(E.FMT_422, 96, 64, profile=3, seed=1), E.Case(E.FMT_4444, 96, 64, profile=4, alpha_bits=8, seed=2),
             E.Case(E.FMT_444, 96, 64, interlaced=1, profile=2, mbs_per_slice=2, seed=3),
             E.Case(E.FMT_4444, 96, 64, interlaced=2, profile=4, alpha_bits=16, seed=4)]
    mem = PU.DevMem()
    works, outs, sizes = [], [], []
    for c in cases:
        ptrs = [mem.put(c.padded(p)) if c.planes[p] is not None else None for p in range(4)]
        o = mem.put(np.zeros(c.capacity(), np.uint8))
        z = mem.put(np.zeros(1, np.int32))
        outs.append(o); sizes.append(z)
        works.append(c.work(ptrs, o, c.capacity(), z))
    arr = (tables.FFProresEncodeWork * len(works))(*works)
    need = gpu.lib.ff_prores_encode_workspace_cuda(arr, len(works))
    ws = mem.put(np.zeros(max(need, 1), np.uint8))
    assert gpu.lib.ff_prores_encode_frames_cuda(arr, len(works), C.c_void_p(ws), need, None) == 0
    mem.sync()
    pkts = []
    for c, o, z in zip(cases, outs, sizes):
        n = int(mem.get(z, np.int32, (1,))[0])
        pkts.append(D.Pkt(mem.get(o, np.uint8, (n,)), c.w, c.h, repr(c)))         # the host copy feeds only the probe and the reference
    D.check(gpu.lib, dref, mem, pkts, dev_pkts=outs)


_pools = {}


def pool(eref, w, h):
    """packets of every format and field order at w x h from the reference encoder"""
    if (w, h) not in _pools:
        _pools[(w, h)] = [D.encode(eref, fmt, w, h, interlaced=il, profile=prof, alpha_bits=ab, seed=k)
                          for k, (fmt, il, prof, ab) in enumerate(((E.FMT_422, 0, 3, 16), (E.FMT_4444, 1, 4, 16), (E.FMT_422, 2, 0, 16),
                                                                   (E.FMT_444, 0, 2, 16), (E.FMT_4444, 0, 4, 8)))]
    return _pools[(w, h)]


@pytest.mark.parametrize("n", [1, 16, 64])
@pytest.mark.parametrize("size", [(1920, 1080), (4096, 2160)])
def test_batches(gpu, dref, eref, n, size):
    p = pool(eref, *size)
    D.check(gpu.lib, dref, PU.DevMem(), [p[k % len(p)] for k in range(n)], pad=64 if n == 16 else 0)


def test_padded_linesizes(gpu, dref, eref):
    pk = [real(eref, n) for n in ("4444_a16", "hq")] + [edited(eref, n) for n in ("bit_flips_alpha", "zero_plane_dc_27")]
    D.check(gpu.lib, dref, PU.DevMem(), pk, pad=48)
    D.check(gpu.lib, dref, PU.DevMem(), pk, pad=2)


def test_refusals(gpu, dref, eref):
    check_refusals(gpu.lib, dref, eref, PU.DevMem())
