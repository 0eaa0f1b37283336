"""The floating-point AAN transforms (ff_faanidct* and ff_faandct / ff_faandct248, libavcodec/faanidct.c and faandct.c) without a GPU:
libav_b200/csrc/faan_dct.cuh through the thread-per-block kernels of faan_idct.cu compiled as host C++ (tests/hostsim/faan_idct_hostsim.cpp),
against the compiled reference (oracle/_ref/libavref.so); the known answers of the reference's own DCT test (tests/golden/fate_dct8x8_faan.txt,
oracle/refbuild/run_faan_selftest.sh); which table entries the hooks fill; and the SASS of the built library: nvcc contracts a * b + c and
may flush denormals, the host build cannot show either, so every kernel that holds a FAAN transform is checked for FFMA, DFMA and .FTZ."""
import ctypes as C
import os
import re
import shutil
import subprocess

import numpy as np
import pytest

from libav_b200 import synth
import hostsim_build

HERE = os.path.dirname(os.path.abspath(__file__))
GOLD = os.path.join(HERE, "golden", "fate_dct8x8_faan.txt")
NB_ITS = 20000
FF_IDCT_FAAN, FF_DCT_FAAN = 20, 6
vp, pd = C.c_void_p, C.c_ssize_t


def P(a, off=0):
    return C.c_void_p(a.ctypes.data + off)


class RefFaan:
    """the reference's five functions, one block per call, on host memory"""

    def __init__(self, lib):
        self.lib = lib
        for name, args in (("ff_faanidct", [vp]), ("ff_faanidct_put", [vp, pd, vp]), ("ff_faanidct_add", [vp, pd, vp]),
                           ("ff_faandct", [vp]), ("ff_faandct248", [vp])):
            getattr(lib, name).restype, getattr(lib, name).argtypes = None, args

    def fdct(self, which, blocks):
        out = np.ascontiguousarray(blocks.copy())
        f = self.lib.ff_faandct if which == 6 else self.lib.ff_faandct248
        for i in range(len(out)):
            f(P(out, 128 * i))
        return out

    def idct(self, mode, blocks, frame=None, off=None, stride=0):
        """mode 0 put / 1 add / 2 in place over copies; returns (blocks, frame)"""
        b = np.ascontiguousarray(blocks.copy())
        f = None if frame is None else frame.copy()
        for i in range(len(b)):
            if mode == 2:
                self.lib.ff_faanidct(P(b, 128 * i))
            else:
                (self.lib.ff_faanidct_put if mode == 0 else self.lib.ff_faanidct_add)(P(f, int(off[i])), stride, P(b, 128 * i))
        return b, f


@pytest.fixture(scope="session")
def fref(built):
    from oracle import loader
    r = loader.ref()
    if r is None:
        pytest.skip("oracle/_ref not built (no reference tree in this environment)")
    return RefFaan(r.lib)


@pytest.fixture
def sim(built):
    lib = hostsim_build.fresh()
    lib.hostsim_faan_fdct.restype, lib.hostsim_faan_fdct.argtypes = C.c_int, [C.c_int, vp, C.c_size_t]
    return lib


# ---------------------------------------------------------------------------------------------------------------------------- cases

def dc_only_blocks():
    """every DC in [-2048, 2047] alone: the IDCT output is DC / 8 everywhere, so DC = 4 (mod 8) lands exactly on .5 (round half to even)"""
    b = np.zeros((4096, 64), np.int16)
    b[:, 0] = np.arange(-2048, 2048)
    return b


def cases():
    r = np.random.default_rng(7)
    full = r.integers(-32768, 32768, size=(600, 64)).astype(np.int16)
    sparse = np.where(r.random((600, 64)) < 0.08, r.integers(-2048, 2048, size=(600, 64)), 0).astype(np.int16)
    single = np.zeros((64, 64), np.int16)
    for i in range(64):
        single[i, 8 * (i % 8):8 * (i % 8) + 8] = r.integers(-1024, 1024, size=8)
    return {"dct0": synth.dct_test_blocks(0, 600), "dct1": synth.dct_test_blocks(1, 600), "dct2": synth.dct_test_blocks(2, 600),
            "full_range": full, "sparse": sparse, "single_row": single, "dc_only": dc_only_blocks()}


def pixel_blocks(n, seed):
    """what the encoder transforms: samples (0..255) and differences (-255..255)"""
    r = np.random.default_rng(seed)
    return np.concatenate([r.integers(0, 256, size=(n, 64)), r.integers(-255, 256, size=(n, 64))]).astype(np.int16)


# ---------------------------------------------------------------------------------------------------------------------------- IDCT

@pytest.mark.parametrize("name", list(cases()))
def test_hostsim_idct_matches_reference(sim, fref, name):
    """the thread-per-block kernel through ff_faanidct_batch_cuda (host-compiled) against the reference: every mode, fused clear, tile- and
    offset-addressed destinations, an odd pitch, blocks at a 2-byte offset"""
    blocks = cases()[name]
    n, tpr = len(blocks), 37
    stride = tpr * 8 + 5
    rows = (n + tpr - 1) // tpr * 8
    frame = np.random.default_rng(1).integers(0, 256, size=(rows, stride), dtype=np.uint8)
    off = np.array([(i // tpr) * 8 * stride + (i % tpr) * 8 for i in range(n)], np.uint32)
    for mode in (0, 1, 2):
        want_b, want_f = fref.idct(mode, blocks, None if mode == 2 else frame, off, stride)
        for clear, use_off in ((0, False), (1, True)):
            raw = np.zeros(n * 64 + 8, np.int16)
            b = raw[1:1 + n * 64].reshape(n, 64); b[:] = blocks
            f = frame.copy()
            assert sim.ff_faanidct_batch_cuda(mode, b.ctypes.data, f.ctypes.data, off.ctypes.data if use_off else None, stride, n,
                                              0 if use_off else tpr, clear, None) == 0
            if mode == 2:
                assert np.array_equal(b, want_b), (name, clear, use_off, np.argwhere(b != want_b)[:4].tolist())
            else:
                assert np.array_equal(f, want_f), (name, mode, clear, use_off)
                assert np.array_equal(b, np.zeros_like(blocks) if clear else blocks)      # put / add leave the coefficients alone
    assert sim.ff_faanidct_batch_cuda(3, None, None, None, 8, 4, 1, 0, None) == -1
    sim.avb200_clear_error()


def test_dc_only_rounds_half_to_even(fref):
    """the reference itself: DC = 4 (mod 8) gives x.5 everywhere, and lrintf takes the even neighbour (this pins what the kernels must do)"""
    b = dc_only_blocks()
    got, _ = fref.idct(2, b)
    dc = b[:, 0].astype(np.int64)
    want = np.round(dc / 8.0).astype(np.int64)                     # numpy rounds half to even
    assert np.array_equal(got.astype(np.int64), np.repeat(want[:, None], 64, axis=1))


def _golden():
    out = {}
    for line in open(GOLD):
        if line.startswith("idct"):
            f = line.split()
            out[f[0]] = dict(kv.split("=") for kv in f[1:])
    return out


def fate_statistics(got, blocks):
    want = synth.ref_idct(blocks.reshape(-1, 8, 8)).reshape(-1, 64).astype(np.int64)
    err = got.astype(np.int64) - want
    return {"ppe": int(np.abs(err).max()), "omse": "%0.8f" % (float((err * err).sum()) / NB_ITS / 64),
            "ome": "%0.8f" % (float(err.sum()) / NB_ITS / 64), "maxout": int(np.abs(got.astype(np.int64)).max())}


def check_fate(stats, test):
    g = _golden()["idct%d" % test]
    assert stats == {"ppe": int(g["ppe"]), "omse": g["omse"], "ome": g["ome"], "maxout": int(g["maxout"])}, (test, stats, g)


@pytest.mark.parametrize("test", [0, 1, 2])
def test_reference_and_hostsim_reproduce_fate_faani(sim, fref, test):
    blocks = synth.dct_test_blocks(test, NB_ITS)
    got, _ = fref.idct(2, blocks)
    check_fate(fate_statistics(got, blocks), test)
    b = blocks.copy()
    assert sim.ff_faanidct_batch_cuda(2, b.ctypes.data, None, None, 0, len(b), 0, 0, None) == 0
    check_fate(fate_statistics(b, blocks), test)


# ---------------------------------------------------------------------------------------------------------------------------- FDCT

@pytest.mark.parametrize("which", [6, 7])
def test_hostsim_fdct_matches_reference(sim, fref, which):
    """ff_faandct / ff_faandct248 (the kernel behind ff_fdct_batch_cuda 6 / 7, host-compiled) against the reference, on pixel blocks and on
    every IDCT case, full-range int16 included (the int16 store wraps like the C code's)"""
    blocks = np.concatenate([pixel_blocks(500, 3 + which)] + list(cases().values()))
    raw = np.zeros(len(blocks) * 64 + 8, np.int16)
    b = raw[1:1 + len(blocks) * 64].reshape(-1, 64); b[:] = blocks
    assert sim.hostsim_faan_fdct(which, b.ctypes.data, len(b)) == 0
    want = fref.fdct(which, blocks)
    assert np.array_equal(b, want), np.argwhere(b != want)[:4].tolist()
    assert sim.hostsim_faan_fdct(5, b.ctypes.data, 1) == -1
    sim.avb200_clear_error()


# ---------------------------------------------------------------------------------------------------------------------------- tables

WORD = C.sizeof(C.c_void_p)


def words(table, nbytes=None):
    n = (nbytes or C.sizeof(table)) // WORD
    return [1 if v else 0 for v in (C.c_void_p * n).from_buffer(table)]


def ref_words(refo, kind, a, b):
    out = np.zeros(64, np.uint8)
    n = refo.table_fill(kind, a, b, out.ctypes.data, len(out))
    assert n > 0
    return out[:n].tolist()


def test_hooks_fill_what_the_reference_fills(built, refo):
    """FDCTDSPContext at dct_algo FF_DCT_FAAN and IDCTDSPContext at idct_algo FF_IDCT_FAAN: exactly the reference's entries at 8 and 10 bit
    (10 bit keeps the 10-bit islow pair / simple IDCT whatever the algorithm says); 9 and 12 bit are left untouched"""
    import libav_b200._lib as L
    from libav_b200 import tables
    lib = L.lib
    for bits in (8, 10):
        t = tables.FDCTDSPContext(); lib.ff_fdctdsp_init_cuda(C.byref(t), FF_DCT_FAAN, bits, int(bits > 8))
        assert words(t) == ref_words(refo, 8, bits, FF_DCT_FAAN), bits
        t = tables.IDCTDSPContext(); lib.ff_idctdsp_init_cuda(C.byref(t), FF_IDCT_FAAN, bits, int(bits > 8))
        assert words(t, 6 * WORD) == ref_words(refo, 10, bits, FF_IDCT_FAAN), bits
        assert t.perm_type == 0 and list(t.idct_permutation) == list(range(64))
    for bits in (9, 12):
        t = tables.FDCTDSPContext(); lib.ff_fdctdsp_init_cuda(C.byref(t), FF_DCT_FAAN, bits, 1)
        assert not any(words(t))
        t = tables.IDCTDSPContext(); lib.ff_idctdsp_init_cuda(C.byref(t), FF_IDCT_FAAN, bits, 1)
        assert not any(words(t))


def test_ff_dct_faan_slots_are_not_the_islow_ones(built):
    import libav_b200._lib as L
    from libav_b200 import tables
    a, b = tables.FDCTDSPContext(), tables.FDCTDSPContext()
    L.lib.ff_fdctdsp_init_cuda(C.byref(a), FF_DCT_FAAN, 8, 0)
    L.lib.ff_fdctdsp_init_cuda(C.byref(b), 0, 8, 0)
    assert words(a) == [1, 1] and (C.c_void_p * 2).from_buffer(a)[:] != (C.c_void_p * 2).from_buffer(b)[:]


# ---------------------------------------------------------------------------------------------------------------------------- SASS

def _sass_functions(obj):
    cuobjdump = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    if not os.path.exists(cuobjdump):
        pytest.skip("cuobjdump not available")
    out = subprocess.run([cuobjdump, "-sass", obj], capture_output=True, text=True, check=True).stdout
    funcs, cur = {}, None
    for line in out.splitlines():
        m = re.match(r"\s+Function : (\S+)", line)
        if m:
            cur = m.group(1); funcs[cur] = []
        elif cur and re.match(r"\s+/\*[0-9a-f]{4,}\*/", line):
            funcs[cur].append(re.sub(r"^@!?U?P\w+\s+", "", line.split("*/", 1)[1].split(";")[0].strip()))      # without the predicate
    return funcs


def test_faan_kernels_are_not_contracted_and_keep_denormals(built):
    """every FAAN kernel of the built library: no FFMA / DFMA (contracted products, which the C code does not have) and no .FTZ (flushed
    denormals).  The one .FTZ instruction nvcc emits for an unsigned integer division (F2I.FTZ.U32.TRUNC of a reciprocal estimate, in the tile
    addressing) is integer arithmetic and is allowed."""
    objdir = os.path.join(os.path.dirname(HERE), "libav_b200", "csrc", "build")
    found = {}
    for obj, pat in (("idctdsp.o", "faan_idct_kernel"), ("faan_idct.o", "faan_"), ("me_cmp.o", "pixblock_kernelILi[67]E|me_cmp_dct_kernel"),
                     ("mpv_quant.o", "mpv_quant_kernelILi6E"), ("me_cmp_enc.o", "me_cmp_enc_kernel")):
        path = os.path.join(objdir, obj)
        assert os.path.exists(path), path
        for name, ins in _sass_functions(path).items():
            if not re.search(pat, name):
                continue
            found[name] = len(ins)
            bad = [i for i in ins if re.search(r"\bFFMA\b|\bDFMA\b|\bFFMA\.|\bDFMA\.", i) or (".FTZ" in i and not i.startswith("F2I.FTZ.U32.TRUNC"))]
            assert not bad, (name, bad[:4])
            assert any(i.startswith("DMUL") for i in ins), name                  # the double products are there
    # staged put / add / in place + 14 fused; fallback + 2 fdct; 2 pixblock + dct_sad / dct_max; 2 quantisers; quant_psnr / bit / rd
    assert len(found) == 19 + 3 + 3 + 2 + 1, sorted(found)
