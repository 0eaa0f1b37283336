"""GPU: ff_mpv_dct_quantize_batch_cuda and the dct_quantize slots against the checker -- the reference's own quantisers
(oracle/_ref/libmpvqref.so) where they travelled, else the plain-C port (oracle/port/orc_mpvq.c), which the CPU suite pins to the reference.
Every state of the CPU suite; n = 1, 37, 65537 and sixteen 1080p 4:2:0 pictures (783,360 blocks) in one call; both quantisers, fused from
pixels and from staged blocks (bitwise equal); per-block qscale over all 31 values; the noise-reduction sums of a whole picture against the
reference's sequential sums; the slots on a live context; guard words around every buffer; a created stream; refusals leave the device
buffers as they were.  Blocks whose reference result reads trellis table entries the reference never writes (undefined there) are left out
of the comparisons with the reference, and counted; the product itself is deterministic on them (fused = staged, created stream = default)."""
import ctypes as C

import numpy as np
import pytest

import mpv_quant_cases as M
import test_mpv_quant_cpu as CPU

pytestmark = pytest.mark.gpu

GUARD = 64                          # guard bytes on each side of every output buffer


@pytest.fixture(scope="session")
def mats(built):
    return M.matrices_checker()


class Guarded:
    """a device buffer with GUARD bytes of a fixed pattern on each side"""

    def __init__(self, a):
        from libav_b200 import device
        a = np.ascontiguousarray(a)
        self.dtype, self.shape, self.nbytes = a.dtype, a.shape, a.nbytes
        host = np.full(a.nbytes + 2 * GUARD, 0xC5, np.uint8)
        host[GUARD:GUARD + a.nbytes] = a.view(np.uint8).reshape(-1)
        self.buf = device.DevBuf.from_numpy(host)
        self.ptr = self.buf.ptr + GUARD

    def get(self):
        raw = self.buf.download(np.uint8, (self.nbytes + 2 * GUARD,))
        assert (raw[:GUARD] == 0xC5).all() and (raw[GUARD + self.nbytes:] == 0xC5).all(), "guard words overwritten"
        return raw[GUARD:GUARD + self.nbytes].view(self.dtype).reshape(self.shape)


def run_gpu(gpu, st, vlc, trellis, recs, blocks=None, pix=None, nr=None, stream=None):
    """the product on the GPU; blocks (n, 64) staged spatial samples, or pix = (cur, ref or None, off, stride) fetched by the kernel.
    Returns (levels, last_index, coded_score) and updates nr in place."""
    from libav_b200 import device
    lib = gpu.lib
    n = len(recs)
    h = lib.ff_mpv_quant_state_cuda(C.byref(st), C.byref(vlc.product()) if vlc else None)
    assert h, gpu.last_error()
    try:
        d_blk = Guarded(np.zeros((n, 64), np.int16) if blocks is None else np.ascontiguousarray(blocks, np.int16))
        d_last = Guarded(np.full(n, -7, np.int32))
        d_score = Guarded(np.full(n, M.SCORE_UNSET, np.int32))
        d_rec = device.DevBuf.from_numpy(np.ascontiguousarray(recs))
        keep = [d_rec]
        if pix is None:
            args = (None, None, None, None, 0)
        else:
            cur, ref, off, stride = pix
            d_cur, d_off = device.DevBuf.from_numpy(cur), device.DevBuf.from_numpy(off)
            d_ref = device.DevBuf.from_numpy(ref) if ref is not None else None
            keep += [d_cur, d_off, d_ref]
            args = (d_cur.ptr, d_ref.ptr if d_ref else None, d_off.ptr, None, stride)
        nrs = None
        if nr:
            d_o, d_s, d_c = Guarded(nr.offset), Guarded(nr.sum), Guarded(nr.count)
            nrs = M.nr_struct(d_o.ptr, d_s.ptr, d_c.ptr)
        gpu.check(lib.ff_mpv_dct_quantize_batch_cuda(h, trellis, d_rec.ptr, *args, d_blk.ptr, n, d_last.ptr, d_score.ptr,
                                                     C.byref(nrs) if nr else None, stream), "ff_mpv_dct_quantize_batch_cuda")
        device.sync()
        if nr:
            assert np.array_equal(d_o.get(), nr.offset)
            nr.sum[:], nr.count[:] = d_s.get(), d_c.get()
        return d_blk.get(), d_last.get(), d_score.get()
    finally:
        lib.ff_mpv_quant_state_free_cuda(h)


def test_every_state_both_quantisers(gpu, mats):
    chk = M.checker()
    skipped = 0
    for label, st, vlc, trellis, recs, blk, nr in CPU._cases(mats, n=2000, seed=3):
        nr1, nr2 = (nr.copy(), nr.copy()) if nr else (None, None)
        want = chk.run(st, vlc, trellis, recs, blk, nr1)
        skip = M.undefined_blocks(st, vlc, trellis, recs, blk, nr)
        skipped += int(skip.sum())
        M.compare(label, want, *run_gpu(gpu, st, vlc, trellis, recs, blocks=blk, nr=nr2), trellis, skip=skip)
        if nr:
            assert np.array_equal(nr1.sum, nr2.sum) and np.array_equal(nr1.count, nr2.count), label
    assert skipped < 2000


@pytest.mark.parametrize("n", [1, 37, 65537])
def test_sizes_fused_and_staged(gpu, mats, n):
    """n blocks with every qscale: the fused front end (diff_pixels and get_pixels) equals the staged path bitwise, and both equal the checker"""
    chk = M.checker()
    for label, st in M.states(mats)[:: 5 if n > 1000 else 2]:
        vlc = M.Vlc(8)
        cur, rf, off, stride = M.planes(n, 21 + n)
        recs = M.records(n, 22 + n)
        for trellis in (0, 1):
            for inter in (True, False):
                blk = M.spatial(cur, rf, off, stride, inter=inter)
                skip = M.undefined_blocks(st, vlc, trellis, recs, blk)
                staged = run_gpu(gpu, st, vlc, trellis, recs, blocks=blk)
                fused = run_gpu(gpu, st, vlc, trellis, recs, pix=(cur, rf if inter else None, off, stride))
                for a, b in zip(staged, fused):                  # (bitwise, the blocks the reference leaves undefined included)
                    assert np.array_equal(a, b), (label, trellis, inter)
                M.compare((label, n, trellis, inter), chk.run(st, vlc, trellis, recs, blk), *fused, trellis, skip=skip)


def hd_pictures(n_pic, seed):
    """n_pic 1080p 4:2:0 pictures (1920 x 1088 luma) as one plane: per picture 1088 luma rows, then 544 rows holding Cb | Cr side by side.
    A smooth picture with texture and noise, and a prediction that differs from it by a small motion-like error.  Returns cur, ref, off,
    stride and the chroma flag per block (macroblock order: 4 luma blocks, Cb, Cr)."""
    rng = np.random.default_rng(seed)
    W, H, stride = 1920, 1088, 1920
    rows = n_pic * (H + H // 2)
    y, x = np.arange(rows, dtype=np.float32), np.arange(stride, dtype=np.float32)
    base = (128 + 60 * np.outer(np.cos(y / 23), np.sin(x / 37)) + 40 * np.outer(np.cos(y / 13), np.sin(x / 11))).astype(np.int16)
    cur = np.clip(base + rng.integers(-20, 21, base.shape, dtype=np.int16), 0, 255).astype(np.uint8)
    ref = np.clip(base + rng.integers(-6, 7, base.shape, dtype=np.int16), 0, 255).astype(np.uint8)
    del base
    mbw, mbh = W // 16, H // 16
    offs, chroma = [], []
    for p in range(n_pic):
        y0 = p * (H + H // 2)
        for my in range(mbh):
            for mx in range(mbw):
                for b in range(4):
                    offs.append((y0 + my * 16 + 8 * (b >> 1)) * stride + mx * 16 + 8 * (b & 1)); chroma.append(0)
                for c in range(2):
                    offs.append((y0 + H + my * 8) * stride + c * (W // 2) + mx * 8); chroma.append(1)
    return cur, ref, np.array(offs, np.uint32), stride, np.array(chroma, bool)


def test_sixteen_1080p_pictures(gpu, mats):
    """783,360 blocks in one call, per-macroblock qscale over all 31 values, intra and inter macroblocks, both quantisers"""
    chk = M.checker()
    cur, rf, off, stride, chroma = hd_pictures(16, 5)
    n = len(off)
    assert n == 783360
    rng = np.random.default_rng(6)
    recs = np.zeros(n, M.REC)
    mb = np.arange(n) // 6
    q = rng.integers(1, 32, n // 6 + 1)
    intra = rng.random(n // 6 + 1) < 0.2
    lam = (q.astype(np.int64) ** 2 * 128 * 109 // 128).astype(np.uint32)
    recs["qscale"], recs["intra"], recs["chroma"], recs["lambda2"] = q[mb], intra[mb], chroma, lam[mb]
    recs["dc_scale"] = 8
    st = M.make_state(mats, 0, M.FMT_H263, maxq=127, elim=(3, 4), seed=99)
    vlc = M.Vlc(9)
    blk = M.spatial(cur, rf, off, stride)
    for trellis in (0, 1):
        got = run_gpu(gpu, st, vlc, trellis, recs, pix=(cur, rf, off, stride))
        M.compare(("1080p x16", trellis), chk.run(st, vlc, trellis, recs, blk), *got, trellis,
                  skip=M.undefined_blocks(st, vlc, trellis, recs, blk))


def test_noise_reduction_sums_of_a_picture(gpu, mats):
    """one 1080p picture with noise reduction: the device's atomically added sums equal the reference's sequential ones"""
    chk = M.checker()
    cur, rf, off, stride, chroma = hd_pictures(1, 7)
    n = len(off)
    recs = M.records(n, 8)
    recs["chroma"] = chroma
    st = M.make_state(mats, 2, M.FMT_MPEG1, matrices="random", seed=98)
    blk = M.spatial(cur, rf, off, stride)
    for trellis in (0, 1):
        nr1, nr2 = M.NR(3), M.NR(3)
        want = chk.run(st, M.Vlc(10), trellis, recs, blk, nr1)
        got = run_gpu(gpu, st, M.Vlc(10), trellis, recs, pix=(cur, rf, off, stride), nr=nr2)
        M.compare(("nr", trellis), want, *got, trellis, skip=M.undefined_blocks(st, M.Vlc(10), trellis, recs, blk, M.NR(3)))
        assert np.array_equal(nr1.sum, nr2.sum) and np.array_equal(nr1.count, nr2.count)
        assert nr2.count.sum() - M.NR(3).count.sum() == n


def test_created_stream_gives_default_stream_result(gpu, mats):
    st = M.make_state(mats, 0, M.FMT_MPEG1, seed=97)
    cur, rf, off, stride = M.planes(5000, 30)
    recs = M.records(5000, 31)
    s = gpu.lib.avb200_stream_create()
    assert s
    try:
        for trellis in (0, 1):
            a = run_gpu(gpu, st, M.Vlc(11), trellis, recs, pix=(cur, rf, off, stride))
            b = run_gpu(gpu, st, M.Vlc(11), trellis, recs, pix=(cur, rf, off, stride), stream=s)
            for x, y in zip(a, b):
                assert np.array_equal(x, y)
    finally:
        gpu.lib.avb200_stream_destroy(s)


def test_slots_on_a_live_context(gpu, mats):
    assert CPU.slot_cases(gpu.lib, mats) > 1000
    CPU.hook_refusals(gpu.lib, mats)


def test_refusals_leave_device_buffers(gpu, mats):
    from libav_b200 import device
    keep = []

    def upload(a):
        b = device.DevBuf.from_numpy(np.ascontiguousarray(a))
        keep.append(b)
        return b.ptr

    def download(p, like):
        b = next(k for k in keep if k.ptr == p)
        return b.download(like.dtype, like.shape)

    CPU.batch_refusals(gpu.lib, upload, download, mats)
