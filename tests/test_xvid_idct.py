"""The Xvid IDCT (ff_xvid_idct / xvid_idct_put / xvid_idct_add, libavcodec/xvididct.c), what ff_xvid_idct_init() installs for MPEG-4 streams
written by Xvid: libav_b200/csrc/xvid_idct.cuh + xvid_idct.cu + the Xvid instance of the 8-bit IDCT kernel in idctdsp.cu.

CPU: the oracle port (oracle/port/orc_xvid.c) against the compiled reference (oracle/_ref/libxvidref.so) and against the known answers of the
reference's own IDCT test (tests/golden/fate_idct8x8_xvid.txt, oracle/refbuild/run_xvid_selftest.sh); which table entries
ff_xvid_idct_init_cuda fills; the thread-per-block kernel and the slots compiled as host C++ (tests/hostsim/xvid_idct_hostsim.cpp).
GPU: ff_xvid_idct_batch_cuda, ff_mpeg_dequant_xvid_idct_batch_cuda and the slots byte for byte against the checker."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

from libav_b200 import synth

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
GOLD = os.path.join(HERE, "golden", "fate_idct8x8_xvid.txt")
XVID_REF = os.path.join(ROOT, "oracle", "_ref", "libxvidref.so")
NB_ITS = 20000
FF_IDCT_AUTO, FF_IDCT_INT, FF_IDCT_SIMPLE, FF_IDCT_XVID, FF_IDCT_FAAN = 0, 1, 2, 14, 20
vp, pd, sz, i32 = C.c_void_p, C.c_ssize_t, C.c_size_t, C.c_int


def P(a, off=0):
    return C.c_void_p(a.ctypes.data + off)


class Xvid:
    """one implementation of the Xvid IDCT on host memory: the compiled reference (prefix ref_) or the port (prefix orc_)"""

    def __init__(self, lib, prefix):
        self.lib, self.prefix = lib, prefix
        for name, args in (("xvid_idct_put", [vp, pd, vp]), ("xvid_idct_add", [vp, pd, vp]), ("xvid_idct", [vp])):
            f = getattr(lib, prefix + name)
            f.restype, f.argtypes = None, args
            setattr(self, name, f)
        self._batch = getattr(lib, prefix + "xvid_idct_batch")
        self._batch.restype = None
        self._batch.argtypes = [i32, vp, vp, vp, pd, sz] + ([i32] if prefix == "orc_" else [])

    def batch(self, mode, blocks, frame, off, stride):
        """mode 0 put / 1 add / 2 in place over copies; returns (blocks, frame)"""
        b = np.ascontiguousarray(blocks.copy())
        f = None if frame is None else frame.copy()
        extra = (os.cpu_count() or 1,) if self.prefix == "orc_" else ()
        self._batch(mode, P(b), None if f is None else P(f), None if off is None else P(off), stride, len(b), *extra)
        return b, f


@pytest.fixture(scope="session")
def xport(built):
    from oracle import loader
    return Xvid(loader.port().lib, "orc_")


@pytest.fixture(scope="session")
def xref(built):
    if not os.path.exists(XVID_REF):
        pytest.skip("oracle/_ref not built (no reference tree in this environment)")
    lib = C.CDLL(XVID_REF)
    lib.ref_xvid_table_fill.restype = i32
    lib.ref_xvid_table_fill.argtypes = [i32, i32, vp, vp, vp]
    return Xvid(lib, "ref_")


@pytest.fixture(scope="session")
def xchk(built):
    """the strongest Xvid checker available: the compiled reference if it travelled, else the port"""
    from oracle import loader
    return Xvid(C.CDLL(XVID_REF), "ref_") if os.path.exists(XVID_REF) else Xvid(loader.port().lib, "orc_")


# ---------------------------------------------------------------------------------------------------------------------------- cases

def sparse_blocks(n, seed):
    """rows drawn from the shapes that select each branch of idct_row (DC only, DC + in[1..3], DC + in[4], in[5..7] only, everything,
    nothing), with the last five / four rows often all zero so that ff_xvid_idct picks idct_col_3 / idct_col_4 as well as idct_col_8"""
    r = np.random.default_rng(seed)
    out = np.zeros((n, 8, 8), np.int16)
    for i in range(n):
        tail = r.integers(0, 3)                       # 0: rows 3.. zero (col_3), 1: rows 4.. zero (col_4), 2: anything (col_8)
        for y in range(8):
            if (tail == 0 and y >= 3) or (tail == 1 and y >= 4):
                continue
            shape = r.integers(0, 6)
            row = np.zeros(8, np.int64)
            if shape in (0, 1, 2, 4):
                row[0] = r.integers(-1024, 1024)
            if shape == 1:
                row[1:4] = r.integers(-300, 300, 3) * r.integers(0, 2, 3)
            if shape == 2:
                row[4] = r.integers(-300, 300)
            if shape == 3:
                row[5:8] = r.integers(-300, 300, 3)
            if shape == 4:
                row[1:8] = r.integers(-300, 300, 7)
            out[i, y] = row
    return out.reshape(n, 64)


def dc_minus4_blocks():
    """row 0 = {-4, 0, ...} (idct_row returns 0 and leaves it as it was), and that block with one more non-zero coefficient anywhere"""
    out = [np.zeros(64, np.int16)]
    out[0][0] = -4
    for pos in range(1, 64):
        for v in (1, -1, 37):
            b = out[0].copy(); b[pos] = v; out.append(b)
    for dc in (-5, -3, -4 - 8, 0):
        b = np.zeros(64, np.int16); b[0] = dc; out.append(b)
    return np.array(out, np.int16)


def cases():
    rng = np.random.default_rng(7)
    return {
        "dct0": synth.dct_test_blocks(0, 4096), "dct1": synth.dct_test_blocks(1, 4096), "dct2": synth.dct_test_blocks(2, 4096),
        "sparse": sparse_blocks(3000, 3), "dc_minus4": dc_minus4_blocks(),
        "full_range": rng.integers(-32768, 32768, size=(2048, 64)).astype(np.int16),
        "pm2048": rng.integers(-2048, 2048, size=(2048, 64)).astype(np.int16), "dense": synth.dense_blocks(2048, seed=4),
    }


def frame_for(n, stride, seed):
    return np.random.default_rng(seed).integers(0, 256, size=(n * 8, abs(stride)), dtype=np.uint8)


# ---------------------------------------------------------------------------------------------------------------------------- CPU

@pytest.mark.parametrize("name", list(cases()))
def test_port_matches_reference(xport, xref, name):
    """the formula-wise restatement equals the unmodified xvididct.c block for block: in place, and put / add with clamping at a positive and
    a negative line size"""
    blocks = cases()[name]
    n = len(blocks)
    a, _ = xport.batch(2, blocks, None, None, 0)
    b, _ = xref.batch(2, blocks, None, None, 0)
    assert np.array_equal(a, b), (name, np.flatnonzero((a != b).any(axis=1))[:5])
    for stride in (8, -8):
        frame = frame_for(n, 8, 5)
        # block i's top row at i * 64 (positive line size) or at its bottom row (negative: the 8 x 8 runs upwards)
        off = (np.arange(n, dtype=np.uint32) * 64 + (0 if stride > 0 else 56)).astype(np.uint32)
        for mode in (0, 1):
            _, fa = xport.batch(mode, blocks, frame, off, stride)
            _, fb = xref.batch(mode, blocks, frame, off, stride)
            assert np.array_equal(fa, fb), (name, mode, stride)


def _golden():
    out = {}
    for line in open(GOLD):
        if line.startswith("test"):
            f = line.split()
            out[int(f[0][4:])] = dict(kv.split("=") for kv in f[1:])
    return out


def fate_statistics(got, blocks):
    want = synth.ref_idct(blocks.reshape(-1, 8, 8)).reshape(-1, 64).astype(np.int64)
    err = got.astype(np.int64) - want
    return {"ppe": int(np.abs(err).max()), "omse": "%0.8f" % (float((err * err).sum()) / NB_ITS / 64),
            "ome": "%0.8f" % (float(err.sum()) / NB_ITS / 64), "maxout": int(np.abs(got.astype(np.int64)).max())}


def check_fate(stats, test):
    g = _golden()[test]
    # dct.c marks XVID nonspec: the IEEE-1180 thresholds are not asserted (ome of tests 1 and 2 is above 0.0015)
    assert stats == {"ppe": int(g["ppe"]), "omse": g["omse"], "ome": g["ome"], "maxout": int(g["maxout"])}, (test, stats, g)


@pytest.mark.parametrize("test", [0, 1, 2])
def test_port_reproduces_fate_idct8x8_xvid(xport, test):
    blocks = synth.dct_test_blocks(test, NB_ITS)
    got, _ = xport.batch(2, blocks, None, None, 0)
    check_fate(fate_statistics(got, blocks), test)


def _words(t, n=6):
    return [1 if v else 0 for v in (C.c_void_p * n).from_buffer(t)]


def test_table_fill_matches_reference(xref):
    """ff_xvid_idct_init_cuda on a zeroed table fills exactly the entries the reference's ff_xvid_idct_init fills, and where it fills them
    perm_type FF_IDCT_PERM_NONE and the identity permutation"""
    import libav_b200._lib as L
    from libav_b200 import tables
    n = 0
    for algo in (FF_IDCT_AUTO, FF_IDCT_XVID, FF_IDCT_SIMPLE, FF_IDCT_INT, FF_IDCT_FAAN):
        for bits in (8, 9, 10):
            t = tables.IDCTDSPContext()
            L.lib.ff_xvid_idct_init_cuda(C.byref(t), algo, bits)
            want = np.zeros(6, np.uint8); ptype = C.c_int(-1); perm = np.zeros(64, np.uint8)
            assert xref.lib.ref_xvid_table_fill(bits, algo, P(want), C.byref(ptype), P(perm)) == 6
            assert _words(t) == want.tolist(), (algo, bits)
            if any(want):
                n += 1
                assert t.perm_type == ptype.value == 0 and list(t.idct_permutation) == list(perm) == list(range(64)), (algo, bits)
            else:
                assert t.perm_type == 0 and not any(t.idct_permutation)
    assert n == 2


def test_simple_idct_hook_leaves_xvid_alone(built):
    """ff_idctdsp_init_cuda keeps leaving the transform entries alone for FF_IDCT_XVID (the reference's ff_idctdsp_init installs the simple
    IDCT there; the Xvid transform comes from ff_xvid_idct_init_cuda)"""
    import libav_b200._lib as L
    from libav_b200 import tables
    t = tables.IDCTDSPContext()
    L.lib.ff_idctdsp_init_cuda(C.byref(t), FF_IDCT_XVID, 8, 0)
    assert not any(_words(t)[3:6])


# the host-compiled sources the Xvid library needs: the shim runtime (error channel, scratch pool) of slots_hostsim.cpp, the high-bit-depth
# table hooks that file's slots.cu refers to, and xvid_idct.cu.  Linked with --no-undefined, so a new dependency of those files is a link
# error here rather than a library that fails at load time.
SIM_SOURCES = ("slots_hostsim.cpp", "slots_hbd_hostsim.cpp", "xvid_idct_hostsim.cpp")


@pytest.fixture(scope="session")
def sim(built):
    """the product's xvid_idct.cu as host C++ (tests/hostsim/xvid_idct_hostsim.cpp).  Built into its own library, written under a temporary
    name and renamed into place, so that concurrent test processes never see a half-written file; nothing else under tests/hostsim/ is
    generated or rewritten."""
    hs = os.path.join(HERE, "hostsim")
    csrc = os.path.join(ROOT, "libav_b200", "csrc")
    lib = os.path.join(hs, "libxvid_hostsim.so")
    srcs = [os.path.join(hs, f) for f in SIM_SOURCES]
    deps = srcs + [os.path.join(hs, "shim", "cuda_runtime.h")] + \
        [os.path.join(csrc, f) for f in os.listdir(csrc) if f.endswith((".cu", ".cuh", ".h"))] + \
        [os.path.join(ROOT, "include", f) for f in ("avdsp_b200.h", "avdsp_b200_tables.h")]
    if not os.path.exists(lib) or any(os.path.getmtime(d) > os.path.getmtime(lib) for d in deps):
        tmp = "%s.%d.tmp" % (lib, os.getpid())
        try:
            subprocess.run(["g++", "-O1", "-std=c++17", "-fPIC", "-shared", "-x", "c++", "-DAVB_HOSTSIM", "-I", os.path.join(hs, "shim"), "-I", csrc,
                            "-Wno-unknown-pragmas", "-Wl,--no-undefined", "-o", tmp] + srcs, check=True)
            os.replace(tmp, lib)
        finally:
            if os.path.exists(tmp):
                os.remove(tmp)
    s = C.CDLL(lib)
    s.avb200_last_error.restype = C.c_char_p
    s.ff_xvid_idct_batch_cuda.argtypes = [i32, vp, vp, vp, pd, sz, i32, i32, vp]
    s.ff_xvid_idct_init_cuda.argtypes = [vp, i32, i32]
    return s


def test_hostsim_thread_per_block_kernel(sim, xref):
    """the thread-per-block kernel through ff_xvid_idct_batch_cuda (host-compiled: "device memory" is host memory) against the reference:
    every mode, fused clear, tile- and offset-addressed destinations, an odd pitch, blocks at a 2-byte offset"""
    for name in ("dct0", "sparse", "dc_minus4", "full_range"):
        blocks = cases()[name][:1000]
        n, tpr = len(blocks), 37
        stride = tpr * 8 + 5
        rows = (n + tpr - 1) // tpr * 8
        frame = np.random.default_rng(1).integers(0, 256, size=(rows, stride), dtype=np.uint8)
        off = np.array([(i // tpr) * 8 * stride + (i % tpr) * 8 for i in range(n)], np.uint32)
        for mode in (0, 1, 2):
            want_b, want_f = xref.batch(mode, blocks, None if mode == 2 else frame, None if mode == 2 else off, stride)
            for clear, use_off in ((0, False), (1, True)):
                raw = np.zeros(n * 64 + 8, np.int16)           # blocks at a 2-byte offset
                b = raw[1:1 + n * 64].reshape(n, 64); b[:] = blocks
                f = frame.copy()
                assert sim.ff_xvid_idct_batch_cuda(mode, b.ctypes.data, f.ctypes.data, off.ctypes.data if use_off else None, stride, n,
                                                   0 if use_off else tpr, clear, None) == 0
                if mode == 2:
                    assert np.array_equal(b, want_b), (name, clear, use_off)
                else:
                    assert np.array_equal(f, want_f), (name, mode, clear, use_off)
                    assert np.array_equal(b, np.zeros_like(blocks) if clear else blocks)
    assert sim.ff_xvid_idct_batch_cuda(3, None, None, None, 8, 4, 1, 0, None) == -1
    assert sim.avb200_last_error().decode()
    sim.avb200_clear_error()


def slot_cases(table, xvid, rng, blocks):
    """the three slots of a filled table like a codec calls them, against the checker's: put / add at a positive and a negative line size,
    in place (block compared); returns the number of comparisons"""
    n = 0
    for i, blk in enumerate(blocks):
        for stride in (40, -40):
            for slot, ref in ((table.idct_put, xvid.xvid_idct_put), (table.idct_add, xvid.xvid_idct_add)):
                pix = rng.integers(0, 256, size=(8, 40), dtype=np.uint8)
                a, b = pix.copy(), pix.copy()
                base = 16 if stride > 0 else 7 * 40 + 16
                slot(C.cast(a.ctypes.data + base, C.POINTER(C.c_uint8)), stride, np.ascontiguousarray(blk.copy()).ctypes.data_as(C.POINTER(C.c_int16)))
                ref(P(b, base), stride, P(np.ascontiguousarray(blk.copy())))
                assert np.array_equal(a, b), (i, stride)
                n += 1
        x, y = np.ascontiguousarray(blk.copy()), np.ascontiguousarray(blk.copy())
        table.idct(x.ctypes.data_as(C.POINTER(C.c_int16)))
        xvid.xvid_idct(P(y))
        assert np.array_equal(x, y), i
        n += 1
    return n


def slot_blocks():
    c = cases()
    return np.concatenate([c["dct0"][:40], c["sparse"][:40], c["dc_minus4"][:12], c["full_range"][:20]])


def test_hostsim_slots(sim, xref):
    from libav_b200 import tables
    t = tables.IDCTDSPContext()
    sim.ff_xvid_idct_init_cuda(C.byref(t), FF_IDCT_XVID, 8)
    assert slot_cases(t, xref, np.random.default_rng(2), slot_blocks()) == 112 * 5
    assert sim.avb200_last_error().decode() == ""


# ---------------------------------------------------------------------------------------------------------------------------- GPU

def _h2d(L, ptr, a):
    a = np.ascontiguousarray(a)
    L.check(L.lib.avb200_memcpy_h2d(C.c_void_p(ptr), P(a), a.nbytes, None), "h2d")


def _d2h(L, ptr, dtype, shape):
    out = np.empty(shape, dtype)
    L.check(L.lib.avb200_memcpy_d2h(P(out), C.c_void_p(ptr), out.nbytes, None), "d2h")
    L.check(L.lib.avb200_stream_sync(None), "sync")
    return out


def gpu_batch(L, mode, blocks, frame, off, stride, tpr, clear=0, boff=0, foff=0):
    """ff_xvid_idct_batch_cuda with the blocks `boff` bytes and the frame `foff` bytes into their allocations; returns (blocks, frame)"""
    from libav_b200 import device
    n = len(blocks)
    d_b = device.DevBuf(blocks.nbytes + 64)
    _h2d(L, d_b.ptr + boff, blocks)
    d_f = d_o = None
    if mode != 2:
        d_f = device.DevBuf(frame.nbytes + 64)
        _h2d(L, d_f.ptr + foff, frame)
        if off is not None:
            d_o = device.DevBuf.from_numpy(off)
    L.check(L.lib.ff_xvid_idct_batch_cuda(mode, d_b.ptr + boff, d_f.ptr + foff if d_f else None, d_o.ptr if d_o else None, stride, n,
                                          0 if d_o else tpr, clear, None), "ff_xvid_idct_batch_cuda")
    device.sync()
    return _d2h(L, d_b.ptr + boff, np.int16, blocks.shape), (_d2h(L, d_f.ptr + foff, np.uint8, frame.shape) if d_f else None)


def _layout(n, tpr, stride):
    rows = (n + tpr - 1) // tpr * 8
    off = np.array([(i // tpr) * 8 * stride + (i % tpr) * 8 for i in range(n)], np.uint32) if n < 100000 else \
        ((np.arange(n, dtype=np.uint64) // tpr) * 8 * stride + (np.arange(n, dtype=np.uint64) % tpr) * 8).astype(np.uint32)
    return rows, off


def _check_gpu(gpu, xchk, blocks, mode, clear, use_off, tpr, stride, boff=0, foff=0, tma=0):
    n = len(blocks)
    rows, off = _layout(n, tpr, stride)
    frame = np.random.default_rng(n + mode).integers(0, 256, size=(rows, stride), dtype=np.uint8)
    want_b, want_f = xchk.batch(mode, blocks, None if mode == 2 else frame, None if mode == 2 else off, stride)
    if tma:
        gpu.lib.avb200_set_tuning(b"idct_tma", tma)
    try:
        got_b, got_f = gpu_batch(gpu, mode, blocks, frame, off if use_off else None, stride, tpr, clear, boff, foff)
    finally:
        gpu.lib.avb200_set_tuning(b"idct_tma", 0)
    if mode == 2:
        bad = np.flatnonzero((got_b != want_b).any(axis=1))
        assert not len(bad), (mode, bad[:5])
    else:
        assert np.array_equal(got_f, want_f), (mode, clear, use_off, np.argwhere(got_f != want_f)[:4].tolist())
        assert np.array_equal(got_b, np.zeros_like(blocks) if clear else blocks), (mode, clear)


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(cases()))
@pytest.mark.parametrize("mode", [0, 1, 2])
@pytest.mark.parametrize("clear,use_off", [(0, False), (1, False), (0, True), (1, True)])
def test_gpu_batch_matches_checker(gpu, xchk, name, mode, clear, use_off):
    _check_gpu(gpu, xchk, cases()[name], mode, clear, use_off, tpr=37, stride=37 * 8 + 16)


@pytest.mark.gpu
@pytest.mark.parametrize("n", [1, 31, 33, 1000 + 13])
@pytest.mark.parametrize("mode", [0, 1, 2])
@pytest.mark.parametrize("where", ["aligned", "pitch+4", "blocks+2", "blocks+16", "frame+3", "cp.async"])
def test_gpu_batch_shapes_and_alignment(gpu, xchk, n, mode, where):
    """ragged warps, an 8-byte-unaligned pitch or frame and blocks at a 2-byte offset (thread-per-block kernel), blocks at a 16-byte offset
    and the cp.async fetch on the put path (staged kernel)"""
    blocks = np.concatenate([cases()["sparse"], cases()["dc_minus4"]])[:n]
    tpr = 7 if n > 7 else 1
    stride = tpr * 8 + (4 if where == "pitch+4" else 8)
    for clear, use_off in ((0, False), (1, True)):
        _check_gpu(gpu, xchk, blocks, mode, clear, use_off, tpr, stride, boff={"blocks+2": 2, "blocks+16": 16}.get(where, 0),
                   foff=3 if where == "frame+3" else 0, tma=2 if where == "cp.async" else 0)


@pytest.mark.gpu
@pytest.mark.parametrize("mode", [0, 1, 2])
def test_gpu_batch_full_size(gpu, xchk, mode):
    """bench.py's idct_put size: 2^20 blocks, 1024 tiles per row, every block against the checker; put through TMA and through cp.async"""
    n, tpr = 1 << 20, 1024
    blocks = synth.dense_blocks(n, seed=3)
    blocks[::97] = synth.tile_large(cases()["full_range"], n)[::97]
    for tma in ((0, 2) if mode == 0 else (0,)):
        _check_gpu(gpu, xchk, blocks, mode, 0, False, tpr, tpr * 8, tma=tma)


@pytest.mark.gpu
@pytest.mark.parametrize("clear,use_off", [(0, False), (1, True)])
@pytest.mark.parametrize("kind", range(7))
def test_gpu_dequant_xvid_idct_fused(gpu, xchk, checker, kind, clear, use_off):
    """ff_mpeg_dequant_xvid_idct_batch_cuda against the checker's dequantiser followed by the reference's Xvid put (intra kinds) / add
    (inter kinds, blocks with last_index < 0 skipped): both scans, AIC / AC prediction, full-range levels"""
    from libav_b200 import device
    from test_gpu_mpv import INTER, make_case, oracle_dequant
    n, tpr = 1000 + 13, 37
    for alt, aic in ((0, 0), (1, 1)):
        blocks, rec, t, intra, inter = make_case(checker, kind, n, 60 + kind + 7 * alt, alt, aic, wild=True)
        rows = (n + tpr - 1) // tpr
        stride = tpr * 8 + 24
        frame = np.random.RandomState(3).randint(0, 256, (rows * 8, stride)).astype(np.uint8)
        off = np.array([(i // tpr) * 8 * stride + (i % tpr) * 8 for i in range(n)], np.uint32)
        if use_off:
            off = off[np.random.RandomState(4).permutation(n)]
        deq = oracle_dequant(checker, kind, blocks, rec, intra, inter, alt, aic)
        mode = 1 if kind in INTER else 0
        keep = np.ones(n, bool) if mode == 0 else (rec["last"] >= 0)
        idx = np.flatnonzero(keep)
        _, want = xchk.batch(mode, np.ascontiguousarray(deq[idx]), frame, np.ascontiguousarray(off[idx]), stride)
        d_b, d_r, d_f, d_o = [device.DevBuf.from_numpy(np.ascontiguousarray(a)) for a in (blocks, rec, frame, off)]
        gpu.check(gpu.lib.ff_mpeg_dequant_xvid_idct_batch_cuda(kind, C.byref(t), d_r.ptr, d_b.ptr, d_f.ptr, d_o.ptr if use_off else None, stride, n,
                                                               0 if use_off else tpr, clear, None))
        device.sync()
        got = d_f.download(np.uint8, frame.shape)
        assert np.array_equal(got, want), (kind, alt, np.argwhere(got != want)[:4].tolist())
        after = d_b.download(np.int16, blocks.shape)
        if clear:
            assert not after[idx].any() and np.array_equal(after[~keep], blocks[~keep])
        else:
            assert np.array_equal(after, blocks)


@pytest.mark.gpu
def test_gpu_dequant_xvid_refuses_unaligned_blocks(gpu, checker):
    """the fused call has no thread-per-block fallback: real device buffers with the blocks 2 bytes off the 16-byte grid, or a line size off
    the 8-byte grid, are refused before any launch and left as they were"""
    from libav_b200 import device
    from test_gpu_mpv import make_case
    n, tpr = 64, 8
    blocks, rec, t, _, _ = make_case(checker, 5, n, 1, 0, 0, wild=False)
    d_b, d_r, d_f = device.DevBuf(blocks.nbytes + 64), device.DevBuf.from_numpy(rec), device.DevBuf(8 * 8 * (tpr * 8 + 8) + 64)
    d_f.fill(7)
    _h2d(gpu, d_b.ptr + 2, blocks)
    for boff, stride in ((2, tpr * 8), (0, tpr * 8 + 4)):
        if boff == 0:
            _h2d(gpu, d_b.ptr, blocks)
        assert gpu.lib.ff_mpeg_dequant_xvid_idct_batch_cuda(5, C.byref(t), d_r.ptr, d_b.ptr + boff, d_f.ptr, None, stride, n, tpr, 1, None) == -1
        assert "aligned" in gpu.last_error()
        gpu.lib.avb200_clear_error()
        device.sync()
        assert np.array_equal(_d2h(gpu, d_b.ptr + boff, np.int16, blocks.shape), blocks)
        assert (_d2h(gpu, d_f.ptr, np.uint8, (d_f.nbytes,)) == 7).all()


@pytest.mark.gpu
def test_gpu_slots(gpu, xchk):
    """the table ff_xvid_idct_init_cuda fills, called like a codec calls it (checkasm-style); the in-place block is compared too"""
    from libav_b200 import tables
    t = tables.IDCTDSPContext()
    gpu.lib.ff_xvid_idct_init_cuda(C.byref(t), FF_IDCT_AUTO, 8)
    assert t.perm_type == 0 and list(t.idct_permutation) == list(range(64))
    assert slot_cases(t, xchk, np.random.default_rng(4), slot_blocks()) == 112 * 5
    assert gpu.last_error() == ""


@pytest.mark.gpu
@pytest.mark.parametrize("test", [0, 1, 2])
def test_gpu_reproduces_fate_idct8x8_xvid(gpu, test):
    blocks = synth.dct_test_blocks(test, NB_ITS)
    got, _ = gpu_batch(gpu, 2, blocks, None, None, 0, 0)
    check_fate(fate_statistics(got, blocks), test)
