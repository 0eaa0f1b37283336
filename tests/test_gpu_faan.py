"""The floating-point AAN transforms on the GPU, byte for byte against the compiled reference (oracle/_ref/libavref.so: ff_faanidct*,
ff_faandct, ff_faandct248): ff_faanidct_batch_cuda (staged and thread-per-block paths), ff_mpeg_dequant_faanidct_batch_cuda, the flush's
transform 3, the FF_IDCT_FAAN slots, ff_fdct_batch_cuda / ff_pixblock_fdct_batch_cuda 6 / 7, the FF_DCT_FAAN slots and the FAAN dct_sad /
dct_max of ff_me_cmp_batch_cuda.  There is no plain-C port of these transforms, so the file skips where the reference was not built."""
import ctypes as C

import numpy as np
import pytest

from libav_b200 import synth
from test_faan_cpu import RefFaan, cases, pixel_blocks, fate_statistics, check_fate, NB_ITS, FF_IDCT_FAAN, FF_DCT_FAAN, P

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="session")
def fref(built):
    from oracle import loader
    r = loader.ref()
    if r is None:
        pytest.skip("oracle/_ref not built (no reference tree in this environment)")
    return RefFaan(r.lib)


def _h2d(L, ptr, a):
    a = np.ascontiguousarray(a)
    L.check(L.lib.avb200_memcpy_h2d(C.c_void_p(ptr), P(a), a.nbytes, None), "h2d")


def _d2h(L, ptr, dtype, shape):
    out = np.empty(shape, dtype)
    L.check(L.lib.avb200_memcpy_d2h(P(out), C.c_void_p(ptr), out.nbytes, None), "d2h")
    L.check(L.lib.avb200_stream_sync(None), "sync")
    return out


def _layout(n, tpr, stride):
    rows = (n + tpr - 1) // tpr * 8
    i = np.arange(n, dtype=np.uint64)
    return rows, ((i // tpr) * 8 * stride + (i % tpr) * 8).astype(np.uint32)


def gpu_idct(L, mode, blocks, frame, off, stride, tpr, clear=0, boff=0, foff=0):
    """ff_faanidct_batch_cuda with the blocks `boff` bytes and the frame `foff` bytes into their allocations; returns (blocks, frame)"""
    from libav_b200 import device
    d_b = device.DevBuf(blocks.nbytes + 64)
    _h2d(L, d_b.ptr + boff, blocks)
    d_f = d_o = None
    if mode != 2:
        d_f = device.DevBuf(frame.nbytes + 64)
        _h2d(L, d_f.ptr + foff, frame)
        if off is not None:
            d_o = device.DevBuf.from_numpy(off)
    L.check(L.lib.ff_faanidct_batch_cuda(mode, d_b.ptr + boff, d_f.ptr + foff if d_f else None, d_o.ptr if d_o else None, stride, len(blocks),
                                         0 if d_o else tpr, clear, None), "ff_faanidct_batch_cuda")
    device.sync()
    return _d2h(L, d_b.ptr + boff, np.int16, blocks.shape), (_d2h(L, d_f.ptr + foff, np.uint8, frame.shape) if d_f else None)


def check_idct(gpu, fref, blocks, mode, clear, use_off, tpr, stride, boff=0, foff=0):
    n = len(blocks)
    rows, off = _layout(n, tpr, stride)
    frame = np.random.default_rng(n + mode).integers(0, 256, size=(rows, stride), dtype=np.uint8)
    want_b, want_f = fref.idct(mode, blocks, None if mode == 2 else frame, off, stride)
    got_b, got_f = gpu_idct(gpu, mode, blocks, frame, off if use_off else None, stride, tpr, clear, boff, foff)
    if mode == 2:
        assert np.array_equal(got_b, want_b), (mode, np.flatnonzero((got_b != want_b).any(axis=1))[:5])
    else:
        assert np.array_equal(got_f, want_f), (mode, clear, use_off, np.argwhere(got_f != want_f)[:4].tolist())
        assert np.array_equal(got_b, np.zeros_like(blocks) if clear else blocks), (mode, clear)


@pytest.mark.parametrize("name", list(cases()))
@pytest.mark.parametrize("mode", [0, 1, 2])
@pytest.mark.parametrize("clear,use_off", [(0, False), (1, False), (0, True), (1, True)])
def test_idct_batch(gpu, fref, name, mode, clear, use_off):
    check_idct(gpu, fref, cases()[name], mode, clear, use_off, 37, 37 * 8 + 24)


@pytest.mark.parametrize("n", [1, 31, 33, 1000 + 13])
@pytest.mark.parametrize("mode", [0, 1, 2])
@pytest.mark.parametrize("where", ["aligned", "pitch+4", "blocks+2", "blocks+16", "frame+3"])
def test_idct_shapes_and_alignment(gpu, fref, n, mode, where):
    """the staged kernel (16-byte blocks, 8-byte rows) and the thread-per-block kernel (anything else)"""
    blocks = np.concatenate([cases()["full_range"], cases()["dct1"]])[:n]
    tpr = 13
    stride = tpr * 8 + (4 if where == "pitch+4" else 16)
    boff = {"blocks+2": 2, "blocks+16": 16}.get(where, 0)
    check_idct(gpu, fref, blocks, mode, 0, False, tpr, stride, boff=boff, foff=3 if where == "frame+3" else 0)


@pytest.mark.parametrize("mode", [0, 2])
def test_idct_full_size(gpu, fref, mode):
    """2^20 blocks in one call (many grid-stride iterations per warp)"""
    n = 1 << 20
    blocks = np.tile(np.concatenate([cases()["full_range"], cases()["sparse"], cases()["dc_only"][:848]]), (n // 2048, 1))
    assert len(blocks) == n
    check_idct(gpu, fref, blocks, mode, 0, False, 1024, 1024 * 8)


@pytest.mark.parametrize("test", [0, 1, 2])
def test_reproduces_fate_faani(gpu, test):
    blocks = synth.dct_test_blocks(test, NB_ITS)
    got, _ = gpu_idct(gpu, 2, blocks, None, None, 0, 0)
    check_fate(fate_statistics(got, blocks), test)


@pytest.mark.parametrize("clear,use_off", [(0, False), (1, True)])
@pytest.mark.parametrize("kind", range(7))
def test_dequant_faanidct_fused(gpu, fref, checker, kind, clear, use_off):
    """ff_mpeg_dequant_faanidct_batch_cuda against the checker's dequantiser followed by the reference's FAAN put (intra kinds) / add (inter
    kinds, blocks with last_index < 0 skipped)"""
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
        _, want = fref.idct(mode, np.ascontiguousarray(deq[idx]), frame, np.ascontiguousarray(off[idx]), stride)
        d_b, d_r, d_f, d_o = [device.DevBuf.from_numpy(np.ascontiguousarray(a)) for a in (blocks, rec, frame, off)]
        gpu.check(gpu.lib.ff_mpeg_dequant_faanidct_batch_cuda(kind, C.byref(t), d_r.ptr, d_b.ptr, d_f.ptr, d_o.ptr if use_off else None, stride, n,
                                                              0 if use_off else tpr, clear, None))
        device.sync()
        got = d_f.download(np.uint8, frame.shape)
        assert np.array_equal(got, want), (kind, alt, np.argwhere(got != want)[:4].tolist())
        after = d_b.download(np.int16, blocks.shape)
        if clear:
            assert not after[idx].any() and np.array_equal(after[~keep], blocks[~keep])
        else:
            assert np.array_equal(after, blocks)


def test_dequant_faanidct_refuses_unaligned(gpu, checker):
    from libav_b200 import device
    from test_gpu_mpv import make_case
    n, tpr = 64, 8
    blocks, rec, t, _, _ = make_case(checker, 5, n, 1, 0, 0, wild=False)
    d_b, d_r, d_f = device.DevBuf(blocks.nbytes + 64), device.DevBuf.from_numpy(rec), device.DevBuf(8 * 8 * (tpr * 8 + 8) + 64)
    d_f.fill(7)
    _h2d(gpu, d_b.ptr + 2, blocks)
    assert gpu.lib.ff_mpeg_dequant_faanidct_batch_cuda(5, C.byref(t), d_r.ptr, d_b.ptr + 2, d_f.ptr, None, tpr * 8, n, tpr, 1, None) == -1
    assert "aligned" in gpu.last_error()
    gpu.lib.avb200_clear_error()
    assert np.array_equal(_d2h(gpu, d_b.ptr + 2, np.int16, blocks.shape), blocks)
    assert (_d2h(gpu, d_f.ptr, np.uint8, (d_f.nbytes,)) == 7).all()


def test_idct_slots(gpu, fref):
    """the three entries ff_idctdsp_init_cuda installs for FF_IDCT_FAAN, called like a codec calls them (positive and negative line size)"""
    from libav_b200 import tables
    t = tables.IDCTDSPContext()
    gpu.lib.ff_idctdsp_init_cuda(C.byref(t), FF_IDCT_FAAN, 8, 0)
    assert t.perm_type == 0 and list(t.idct_permutation) == list(range(64))
    rng = np.random.default_rng(4)
    c = cases()
    for blk in np.concatenate([c["dct0"][:20], c["full_range"][:20], c["dc_only"][2044:2056]]):
        for stride in (40, -40):
            for slot, ref in ((t.idct_put, fref.lib.ff_faanidct_put), (t.idct_add, fref.lib.ff_faanidct_add)):
                pix = rng.integers(0, 256, size=(8, 40), dtype=np.uint8)
                a, b = pix.copy(), pix.copy()
                base = 16 if stride > 0 else 7 * 40 + 16
                x = np.ascontiguousarray(blk.copy())
                slot(C.cast(a.ctypes.data + base, C.POINTER(C.c_uint8)), stride, x.ctypes.data_as(C.POINTER(C.c_int16)))
                ref(P(b, base), stride, P(np.ascontiguousarray(blk.copy())))
                assert np.array_equal(a, b) and np.array_equal(x, blk)
        x, y = np.ascontiguousarray(blk.copy()), np.ascontiguousarray(blk.copy())
        t.idct(x.ctypes.data_as(C.POINTER(C.c_int16)))
        fref.lib.ff_faanidct(P(y))
        assert np.array_equal(x, y)
    assert gpu.last_error() == ""


def test_flush_transform_3(gpu, fref, checker):
    """ff_mpv_flush_pictures_cuda with FAAN residual batches on one decoder-shaped plane (line size wider than the picture): intra blocks
    put, inter blocks added, field-DCT blocks at twice the line size, and an h263_intra batch with its inverse quantiser fused"""
    from libav_b200 import device, tables
    from test_gpu_mpv import make_case, oracle_dequant
    mbw, mbh, ls = 22, 18, 22 * 16 + 64
    rng = np.random.default_rng(11)
    plane = rng.integers(0, 256, size=(mbh * 16 + 8, ls), dtype=np.uint8)
    want = plane.copy()
    mbs = rng.permutation(mbw * mbh)
    groups = [mbs[:120], mbs[120:260], mbs[260:330]]
    batches, keep = [], []
    d_plane = device.DevBuf.from_numpy(plane)
    for gi, (mode, field) in enumerate(((0, 0), (1, 1), (0, 0))):
        offs = []
        for mb in groups[gi]:
            x, y = (mb % mbw) * 16, (mb // mbw) * 16
            for k in range(4):
                offs.append((y + (k >> 1) * (1 if field else 8)) * ls + x + (k & 1) * 8)
        off = np.array(offs, np.uint32)
        stride = ls * (2 if field else 1)
        n = len(off)
        if gi < 2:
            blocks = np.concatenate([cases()["dct2"], cases()["sparse"]])[rng.permutation(1200)[:n]]
            _, want = fref.idct(mode, blocks, want, off, stride)
            dq, t, d_r = -1, None, None
        else:
            blocks, rec, t, intra, inter = make_case(checker, 5, n, 9, 0, 0, wild=True)
            _, want = fref.idct(0, oracle_dequant(checker, 5, blocks, rec, intra, inter, 0, 0), want, off, stride)
            dq, d_r = 5, device.DevBuf.from_numpy(rec)
        d_b, d_o = device.DevBuf.from_numpy(np.ascontiguousarray(blocks)), device.DevBuf.from_numpy(off)
        x = tables.FFMpvResidualBatch()
        x.transform, x.dequant, x.mode, x.clear = 3, dq, mode, 1
        x.tables = C.cast(C.pointer(t), C.c_void_p) if t is not None else None
        x.recs = d_r.ptr if d_r else None
        x.blocks, x.frame, x.dst_off, x.stride, x.n = d_b.ptr, d_plane.ptr, d_o.ptr, stride, n
        keep += [d_b, d_o, d_r, t]
        batches.append(x)
    arr = (tables.FFMpvResidualBatch * len(batches))(*batches)
    w = tables.FFMpvPictureWork()
    w.residual, w.n_residual = C.cast(arr, C.c_void_p), len(arr)
    gpu.check(gpu.lib.ff_mpv_flush_pictures_cuda(C.byref(w), None))
    device.sync()
    got = d_plane.download(np.uint8, plane.shape)
    assert np.array_equal(got, want), np.argwhere(got != want)[:4].tolist()
    for d_b in keep[0::4]:
        assert not d_b.download(np.int16, (d_b.nbytes // 2,)).any()           # clear
    arr[0].transform = 2                                                        # not a transform
    assert gpu.lib.ff_mpv_flush_pictures_cuda(C.byref(w), None) == -1
    gpu.lib.avb200_clear_error()


# ---------------------------------------------------------------------------------------------------------------------------- FDCT

@pytest.mark.parametrize("which", [6, 7])
@pytest.mark.parametrize("boff", [0, 2])
def test_fdct_batch(gpu, fref, which, boff):
    """ff_fdct_batch_cuda 6 / 7 on pixel blocks and on clobbered (full-range) input, at a 16- and a 2-byte aligned address"""
    from libav_b200 import device
    blocks = np.concatenate([pixel_blocks(3000, which)] + list(cases().values()))
    d = device.DevBuf(blocks.nbytes + 64)
    _h2d(gpu, d.ptr + boff, blocks)
    gpu.check(gpu.lib.ff_fdct_batch_cuda(which, d.ptr + boff, len(blocks), None))
    device.sync()
    got = _d2h(gpu, d.ptr + boff, np.int16, blocks.shape)
    want = fref.fdct(which, blocks)
    assert np.array_equal(got, want), np.argwhere(got != want)[:4].tolist()


@pytest.mark.parametrize("which", [6, 7])
@pytest.mark.parametrize("diff", [False, True])
@pytest.mark.parametrize("stride", [64, 67])
def test_pixblock_fdct(gpu, fref, which, diff, stride):
    """ff_pixblock_fdct_batch_cuda 6 / 7: get_pixels / diff_pixels then the FAAN transform in one kernel (word and byte loads)"""
    from libav_b200 import device
    rng = np.random.default_rng(which + 2 * diff + stride)
    h = 64
    s1, s2 = rng.integers(0, 256, size=(h, stride), dtype=np.uint8), rng.integers(0, 256, size=(h, stride), dtype=np.uint8)
    n = 400
    ys, xs = rng.integers(0, h - 8, n), rng.integers(0, stride - 8, n)
    if stride == 64:
        xs &= ~7
    off1 = (ys * stride + xs).astype(np.uint32)
    off2 = np.roll(off1, 3)
    blk = np.array([s1[y:y + 8, x:x + 8].astype(np.int16) - (s2[(o // stride):(o // stride) + 8, (o % stride):(o % stride) + 8] if diff else 0)
                    for y, x, o in zip(ys, xs, off2)], np.int16).reshape(n, 64)
    want = fref.fdct(which, blk)
    d1, d2, o1, o2, d_out = (device.DevBuf.from_numpy(a) for a in (s1, s2, off1, off2, np.zeros((n, 64), np.int16)))
    gpu.check(gpu.lib.ff_pixblock_fdct_batch_cuda(which, d1.ptr, d2.ptr if diff else None, o1.ptr, o2.ptr if diff else None, stride, d_out.ptr, n, None))
    device.sync()
    got = d_out.download(np.int16, (n, 64))
    assert np.array_equal(got, want), np.argwhere(got != want)[:4].tolist()


def test_fdct_slots(gpu, fref):
    """the pair ff_fdctdsp_init_cuda installs for FF_DCT_FAAN, called like a codec calls them"""
    from libav_b200 import tables
    t = tables.FDCTDSPContext()
    gpu.lib.ff_fdctdsp_init_cuda(C.byref(t), FF_DCT_FAAN, 8, 0)
    blocks = np.concatenate([pixel_blocks(20, 5), cases()["full_range"][:20]])
    for which, slot in ((6, t.fdct), (7, t.fdct248)):
        want = fref.fdct(which, blocks)
        for i, blk in enumerate(blocks):
            x = np.ascontiguousarray(blk.copy())
            slot(x.ctypes.data_as(C.POINTER(C.c_int16)))
            assert np.array_equal(x, want[i]), (which, i)
    assert gpu.last_error() == ""


@pytest.mark.parametrize("kind", [11, 12])
@pytest.mark.parametrize("sidx,h", [(0, 16), (0, 8), (1, 8)])
def test_me_cmp_dct_metrics_with_faan(gpu, fref, kind, sidx, h):
    """dct_sad / dct_max with dxy 6: diff_pixels -> ff_faandct -> sum / max of |coefficient| per 8x8 quadrant"""
    from libav_b200 import device
    rng = np.random.default_rng(kind + h)
    stride, rows = 96, 64
    cur, ref = rng.integers(0, 256, size=(rows, stride), dtype=np.uint8), rng.integers(0, 256, size=(rows, stride), dtype=np.uint8)
    n = 200
    w = 16 if sidx == 0 else 8
    co = (rng.integers(0, rows - h, n) * stride + rng.integers(0, stride - w, n)).astype(np.uint32)
    ro = (rng.integers(0, rows - h, n) * stride + rng.integers(0, stride - w, n)).astype(np.uint32)
    want = np.zeros(n, np.int64)
    for i in range(n):
        s = 0
        for qy in range(h // 8):
            for qx in range(w // 8):
                a = np.frombuffer(cur.tobytes(), np.uint8)[co[i] + qy * 8 * stride + qx * 8:][:8 * stride].reshape(8, stride)[:, :8]
                b = np.frombuffer(ref.tobytes(), np.uint8)[ro[i] + qy * 8 * stride + qx * 8:][:8 * stride].reshape(8, stride)[:, :8]
                d = fref.fdct(6, (a.astype(np.int16) - b.astype(np.int16)).reshape(1, 64))[0].astype(np.int64)
                s += int(np.abs(d).max()) if kind == 12 else int(np.abs(d).sum())        # the 16-wide slots sum their 8x8 halves
        want[i] = s
    recs = np.zeros(n, [("cur_off", "<u4"), ("ref_off", "<u4")]); recs["cur_off"], recs["ref_off"] = co, ro
    d_c, d_r, d_rec, d_out = (device.DevBuf.from_numpy(a) for a in (cur, ref, recs, np.zeros(n, np.int32)))
    gpu.check(gpu.lib.ff_me_cmp_batch_cuda(kind, sidx, 6, d_c.ptr, d_r.ptr, stride, h, d_rec.ptr, n, d_out.ptr, None))
    device.sync()
    got = d_out.download(np.int32, (n,))
    assert np.array_equal(got.astype(np.int64), want)
