"""TEST INFRASTRUCTURE.  ProRes streams and the work the reference decoder records, for tests/test_prores_cpu.py, tests/test_gpu_prores.py
and tools/prores_bench.py.

Frames are generated from seeds and encoded by the reference's own encoder (oracle/_ref/libproresref.so); decoding them with the
reference records every idct_put call and each picture's slice table, which is what the batch call and the picture call are fed."""
import ctypes as C

import numpy as np

from libav_b200 import tables

vp, i32, pd = C.c_void_p, C.c_int, C.c_ssize_t
FMT_422, FMT_444, FMT_4444 = 0, 1, 2
PROFILES = ("proxy", "lt", "standard", "hq", "4444")


class Rec(C.Structure):        # oracle/refbuild/refapi_prores.c RefProresRec
    _fields_ = [("cap_blocks", C.c_int32), ("cap_slices", C.c_int32), ("blocks", vp), ("qmat", vp), ("dst", vp), ("slice_first", vp),
                ("slice_sf", vp), ("n_blocks", C.c_int32), ("n_slices", C.c_int32), ("n_pics", C.c_int32), ("overflow", C.c_int32),
                ("pic_first_block", C.c_int32 * 2), ("pic_first_slice", C.c_int32 * 2), ("pic_n_slices", C.c_int32 * 2),
                ("pic_num", C.c_int32 * 2), ("frame_type", C.c_int32), ("chroma_factor", C.c_int32), ("mb_width", C.c_int32),
                ("mb_height", C.c_int32), ("slice_width_factor", C.c_int32), ("alpha_info", C.c_int32),
                ("qmat_luma", C.c_uint8 * 64), ("qmat_chroma", C.c_uint8 * 64)]


def ref():
    """the reference's ProRes library with prototypes, or None when oracle/_ref was not built"""
    from oracle import loader
    lib = loader.ref_lib("prores")
    if lib is None:
        return None
    lib.ref_prores_idct_put.restype, lib.ref_prores_idct_put.argtypes = None, [vp, pd, vp, vp]
    lib.ref_prores_dsp_init.restype, lib.ref_prores_dsp_init.argtypes = None, [vp]
    lib.ref_prores_abi.restype, lib.ref_prores_abi.argtypes = None, [vp]
    lib.ref_prores_encode.restype, lib.ref_prores_encode.argtypes = i32, [i32, i32, i32, i32, i32, vp, vp, vp, i32]
    lib.ref_prores_decode.restype, lib.ref_prores_decode.argtypes = i32, [vp, i32, i32, i32, vp, vp, C.POINTER(Rec)]
    return lib


def P(a, off=0):
    return C.c_void_p(a.ctypes.data + off)


# ------------------------------------------------------------------------------------------------------------------------------- blocks

def ref_idct_put(lib, blocks, qmats, qidx):
    """prores_idct_put_c block by block: (final blocks, samples of each block as an (n, 8, 8) uint16 array)"""
    b = np.ascontiguousarray(blocks.copy())
    out = np.zeros((len(b), 8, 8), np.uint16)
    q = np.ascontiguousarray(qmats)
    for i in range(len(b)):
        lib.ref_prores_idct_put(P(out, 128 * i), 16, P(b, 128 * i), P(q, 128 * int(qidx[i])))
    return b, out


def edge_blocks(seed=1):
    """(blocks, qmats, qidx) at the edges of the arithmetic: block * qmat wrapping (to exactly 0 too, which turns a row DC-only), negative
    odd DC values, full-range products that drive both clip bounds, sparse rows, and matrices made as (int16)(qmat * sf) with sf up to 512"""
    r = np.random.default_rng(seed)
    blocks, qm = [], []

    def add(b, q):
        blocks.append(np.asarray(b, np.int64).astype(np.int16).reshape(64)); qm.append(np.asarray(q, np.int64).astype(np.int16).reshape(64))

    ones = np.ones(64)
    for dc in list(range(-41, 42, 2)) + [-32767, -32768, 32767, -1, -3, 1023, -1025]:       # DC-only, odd values: row[0] >> 1 unrounded
        b = np.zeros(64); b[0] = dc; add(b, ones)
    for k in range(64):                                                                        # 256 * 256 wraps to 0: the row turns DC-only
        b = np.zeros(64); b[0] = r.integers(-500, 500); b[k if k else 1] = 256
        q = np.full(64, r.integers(1, 8)); q[k if k else 1] = 256
        add(b, q)
    for _ in range(64):                                                                        # products wrapping to other values
        add(r.integers(-2048, 2048, 64), r.integers(-32768, 32768, 64))
    for _ in range(64):                                                                        # (int16)(qmat byte * sf), sf 1..512
        qb, sf = r.integers(0, 256, 64), int(r.integers(1, 513))
        add(r.integers(-300, 300, 64) * (r.random(64) < 0.2), qb * sf)
    for s in (1, -1):                                                                          # both clip bounds, from every direction
        for _ in range(16):
            add(s * r.integers(20000, 32768, 64), ones * r.integers(1, 4))
    for _ in range(64):                                                                        # sparse rows: DC-only rows next to full ones
        b = np.zeros((8, 8), np.int64)
        for y in range(8):
            kind = r.integers(0, 4)
            if kind == 1: b[y, 0] = r.integers(-4096, 4096)
            if kind == 2: b[y, r.integers(1, 8)] = r.integers(-4096, 4096)
            if kind == 3: b[y] = r.integers(-4096, 4096, 8)
        add(b, r.integers(1, 64, 64))
    full = r.integers(-32768, 32768, (256, 64))                                                # anything at all
    for k in range(256):
        add(full[k], r.integers(-32768, 32768, 64))
    b = np.array(blocks, np.int16)
    return b, np.array(qm, np.int16), np.arange(len(b), dtype=np.uint32)


# ------------------------------------------------------------------------------------------------------------------------------ streams

def source_frame(fmt, w, h, seed):
    """seeded 10-bit planes: smooth gradients plus noise and a few hard edges, (planes, linesizes) with planes[3] alpha or None"""
    r = np.random.default_rng(seed)
    cw = w if fmt != FMT_422 else (w + 1) // 2
    y, x = np.mgrid[0:h, 0:w]

    def plane(pw):
        yy, xx = np.mgrid[0:h, 0:pw]
        base = 512 + 300 * np.sin(xx / (7 + seed % 5) + yy / 11.0) + r.normal(0, 40, (h, pw))
        base[(xx // 24 + yy // 24) % 5 == 0] = r.integers(64, 960)
        return np.ascontiguousarray(np.clip(base, 0, 1023).astype(np.uint16))

    planes = [plane(w), plane(cw), plane(cw), plane(w) if fmt == FMT_4444 else None]
    del x, y
    return planes


def encode(lib, fmt, w, h, interlaced, profile, seed):
    planes = source_frame(fmt, w, h, seed)
    ptrs = (C.c_void_p * 4)(*[p.ctypes.data if p is not None else None for p in planes])
    ls = (C.c_int * 4)(*[p.shape[1] * 2 if p is not None else 0 for p in planes])
    cap = 64 * w * h + (1 << 20)
    out = np.zeros(cap, np.uint8)
    n = lib.ref_prores_encode(fmt, w, h, interlaced, profile, ptrs, ls, P(out), cap)
    assert n > 0, ("encode failed", fmt, w, h, interlaced, profile, n)
    return out[:n].copy()


def scramble(pkt, seed):
    """the same entropy data under other quantisers: both header matrices (any byte, 0 included) and every slice's scale byte are replaced,
    so that qmat * sf reaches 255 * 512 and wraps"""
    r = np.random.default_rng(seed)
    p = pkt.copy()
    hdr = 8
    hsize = int(p[hdr]) << 8 | int(p[hdr + 1])
    assert p[hdr + 19] & 3 == 3, "the encoder writes both matrices"
    p[hdr + 20:hdr + 148] = r.integers(0, 256, 128)
    pos = hdr + hsize
    interlaced = (p[hdr + 12] >> 2) & 3
    for _ in range(2 if interlaced else 1):
        ph = int(p[pos]) >> 3
        size = int.from_bytes(bytes(p[pos + 1:pos + 5]), "big")
        ns = int(p[pos + 5]) << 8 | int(p[pos + 6])
        idx = pos + ph
        data = idx + 2 * ns
        for s in range(ns):
            p[data + 1] = r.choice([1, 2, 100, 128, 129, 200, 224, 255])
            data += int(p[idx + 2 * s]) << 8 | int(p[idx + 2 * s + 1])
        pos += size
    return p


class Frame:
    """a frame buffer for one decoded frame: the four planes (alpha included) in one byte array, each plane with right padding and whole
    macroblocks below, pre-filled with a seeded pattern so that anything written outside the macroblocks would show"""

    def __init__(self, fmt, w, h, interlaced, seed=5):
        self.fmt, self.w, self.h, self.interlaced = fmt, w, h, interlaced
        mbw = (w + 15) // 16
        mbh = 2 * ((h + 31) // 32) if interlaced else (h + 15) // 16
        self.H = 16 * mbh
        cwb = 16 * mbw * (1 if fmt == FMT_422 else 2)                  # chroma plane bytes per line of macroblocks
        self.ls = [32 * mbw + 64, cwb + 32, cwb + 32, 32 * mbw + 64]
        self.off = []
        o = 0
        for p in range(4):
            self.off.append(o)
            o += self.ls[p] * self.H + 64
        self.buf = np.random.default_rng(seed).integers(0, 256, o, dtype=np.uint8)

    def plane(self, buf, p):
        return buf[self.off[p]:self.off[p] + self.ls[p] * self.H]


def decode(lib, frame, pkt, cap_blocks=None):
    """the reference decoder into a copy of frame.buf: (bytes, rec with numpy views: blocks, qmat, dst offsets into the buffer, slices)"""
    out = frame.buf.copy()
    ptrs = (C.c_void_p * 4)(*[out.ctypes.data + frame.off[p] for p in range(4)])
    ls = (C.c_int * 4)(*frame.ls)
    mbw = (frame.w + 15) // 16
    cap_b = cap_blocks or 12 * mbw * (frame.H // 16) + 64
    cap_s = 2 * mbw * (frame.H // 16) + 64
    blocks = np.zeros((cap_b, 64), np.int16); qmat = np.zeros((cap_b, 64), np.int16); dst = np.zeros(cap_b, np.uint64)
    sfirst = np.zeros(cap_s, np.uint32); ssf = np.zeros(cap_s, np.uint16)
    rec = Rec(cap_blocks=cap_b, cap_slices=cap_s, blocks=blocks.ctypes.data, qmat=qmat.ctypes.data, dst=dst.ctypes.data,
              slice_first=sfirst.ctypes.data, slice_sf=ssf.ctypes.data)
    rc = lib.ref_prores_decode(P(pkt), len(pkt), frame.w, frame.h, ptrs, ls, C.byref(rec))
    assert rc == len(pkt) and not rec.overflow, ("decode failed", rc, rec.overflow)
    n = rec.n_blocks
    rec.np_blocks, rec.np_qmat = blocks[:n], qmat[:n]
    rec.np_dst = (dst[:n] - np.uint64(out.ctypes.data)).astype(np.int64)
    rec.np_sfirst, rec.np_ssf = sfirst[:rec.n_slices], ssf[:rec.n_slices]
    return out, rec


def picture_works(frame, rec, base, blocks_ptr_of, slices_ptr_of):
    """one FFProresPictureWork per picture of the decoded frame.  base: the address of the frame buffer the call writes; blocks_ptr_of(k) /
    slices_ptr_of(k): where picture k's coefficients and slice table are"""
    works = []
    il = rec.frame_type != 0
    tff = rec.frame_type == 1
    for k in range(rec.n_pics):
        w = tables.FFProresPictureWork()
        down = il and not (rec.pic_num[k] ^ tff)
        for p in range(3):
            w.data[p] = base + frame.off[p] + (frame.ls[p] if down else 0)
            w.linesize[p] = frame.ls[p] * (2 if il else 1)
            w.mb_rows[p] = frame.H // (32 if il else 16)
        w.mb_width, w.mb_height, w.slice_width_factor, w.chroma_format = rec.mb_width, rec.mb_height, rec.slice_width_factor, rec.chroma_factor
        for i in range(64):
            w.qmat_luma[i] = rec.qmat_luma[i]; w.qmat_chroma[i] = rec.qmat_chroma[i]
        w.slices = slices_ptr_of(k); w.n_slices = rec.pic_n_slices[k]
        w.blocks = blocks_ptr_of(k)
        nb = (rec.pic_first_block[k + 1] if k + 1 < rec.n_pics else rec.n_blocks) - rec.pic_first_block[k]
        w.n_blocks = nb
        works.append(w)
    return works


def slice_table(rec, k):
    """picture k's FFProresSlice array (numpy structured as 2 x uint32 per slice)"""
    s0, ns = rec.pic_first_slice[k], rec.pic_n_slices[k]
    t = np.zeros((ns, 2), np.uint32)
    t[:, 0] = rec.np_sfirst[s0:s0 + ns]
    t[:, 1] = rec.np_ssf[s0:s0 + ns].astype(np.uint32)
    return t


def picture_blocks(rec, k):
    b0 = rec.pic_first_block[k]
    b1 = rec.pic_first_block[k + 1] if k + 1 < rec.n_pics else rec.n_blocks
    return np.ascontiguousarray(rec.np_blocks[b0:b1])


def yuv_equal(frame, a, b):
    """y / u / v planes equal (alpha excluded)"""
    return all(np.array_equal(frame.plane(a, p), frame.plane(b, p)) for p in range(3))


# (fmt, width, height, interlaced 0 / 1 tff / 2 bff, profile): every chroma format, field order and profile, with and without alpha,
# widths whose last slice is 4, 2 or 1 macroblocks (and 4 + 2 + 1), and 1080-line frames
STREAMS = [
    (FMT_422, 192, 64, 0, 3), (FMT_422, 160, 48, 0, 0), (FMT_422, 144, 40, 0, 1), (FMT_422, 112, 32, 0, 2),
    (FMT_422, 176, 64, 1, 3), (FMT_422, 120, 96, 2, 2), (FMT_444, 96, 48, 0, 4), (FMT_444, 184, 40, 1, 4),
    (FMT_4444, 120, 64, 0, 4), (FMT_4444, 72, 80, 2, 4), (FMT_444, 80, 16, 0, 3), (FMT_422, 1920, 1080, 0, 3),
    (FMT_422, 1920, 1080, 1, 1), (FMT_4444, 1920, 1080, 2, 4),
]
SMALL_STREAMS = [s for s in STREAMS if s[2] < 1080]


# ------------------------------------------------------------------------------------------------------------------------- the two calls
class HostMem:
    """'device' memory of the host-compiled library: numpy arrays, addressed directly"""

    def __init__(self):
        self.keep = {}

    def put(self, a, pad=0):
        b = np.zeros(a.nbytes + pad + 16, np.uint8)
        base = (-b.ctypes.data) % 16 + pad                       # 16-byte aligned, then `pad` bytes further
        b[base:base + a.nbytes] = np.ascontiguousarray(a).view(np.uint8).reshape(-1)
        ptr = b.ctypes.data + base
        self.keep[ptr] = b
        return ptr

    def get(self, ptr, dtype, shape):
        b = self.keep[ptr]
        base = ptr - b.ctypes.data
        n = int(np.prod(shape)) * np.dtype(dtype).itemsize
        return b[base:base + n].view(dtype).reshape(shape).copy()

    def sync(self):
        pass


class DevMem:
    """device memory through libav_b200.device.DevBuf"""

    def __init__(self):
        from libav_b200 import device
        self.device, self.keep = device, {}

    def put(self, a, pad=0):
        a = np.ascontiguousarray(a)
        d = self.device.DevBuf(a.nbytes + pad + 256)
        raw = np.zeros(a.nbytes + pad, np.uint8)
        raw[pad:] = a.view(np.uint8).reshape(-1)
        d.upload(raw)
        self.keep[d.ptr + pad] = d
        return d.ptr + pad

    def get(self, ptr, dtype, shape):
        d = self.keep[ptr]
        pad = ptr - d.ptr
        n = int(np.prod(shape)) * np.dtype(dtype).itemsize
        return d.download(np.uint8, pad + n)[pad:].view(dtype).reshape(shape).copy()

    def sync(self):
        self.device.sync()


def run_batch(lib, mem, blocks, qmats, qidx, tiles_per_row=7, pitch_extra=0, block_pad=0, qmat_pad=0, frame_pad=0):
    """ff_prores_idct_put_batch_cuda over blocks laid out as a raster of tiles: (rc, final blocks, samples (n, 8, 8))"""
    n = len(blocks)
    stride = tiles_per_row * 16 + pitch_extra
    rows = (n + tiles_per_row - 1) // tiles_per_row * 8
    i = np.arange(n)
    off = ((i // tiles_per_row) * 8 * stride + (i % tiles_per_row) * 16).astype(np.uint32)
    frame = np.full(rows * stride + 16, 0xee, np.uint8)
    b = mem.put(blocks, block_pad); f = mem.put(frame, frame_pad); o = mem.put(off); q = mem.put(qmats, qmat_pad)
    qi = mem.put(qidx) if qidx is not None else None
    rc = lib.ff_prores_idct_put_batch_cuda(C.c_void_p(b), C.c_void_p(f), C.c_void_p(o), stride, C.c_void_p(q),
                                           None if qi is None else C.c_void_p(qi), n, None)
    mem.sync()
    fb = mem.get(f, np.uint8, frame.shape)
    samples = np.stack([np.frombuffer(np.concatenate([fb[int(off[k]) + y * stride:int(off[k]) + y * stride + 16] for y in range(8)]).tobytes(),
                                      np.uint16).reshape(8, 8) for k in range(n)]) if n else np.zeros((0, 8, 8), np.uint16)
    return rc, mem.get(b, np.int16, blocks.shape), samples


class Decoded:
    """one reference-decoded stream: the frame layout, the reference's output and the recorded work"""

    def __init__(self, lib, spec, seed=3, scrambled=False):
        fmt, w, h, il, prof = spec
        self.spec = spec
        pkt = encode(lib, fmt, w, h, il, prof, seed)
        if scrambled:
            pkt = scramble(pkt, seed)
        self.frame = Frame(fmt, w, h, il, seed)
        self.want, self.rec = decode(lib, self.frame, pkt)


def spread_slices(blocks, table, gap, seed=0):
    """the coefficient buffer re-laid with `gap` blocks of noise in front of every slice (which no slice covers) and the table to match"""
    r = np.random.default_rng(seed)
    firsts = [int(f) for f in table[:, 0]] + [len(blocks)]
    parts, t = [], table.copy()
    pos = 0
    for k in range(len(table)):
        parts.append(r.integers(-32768, 32768, (gap, 64)).astype(np.int16))
        pos += gap
        t[k, 0] = pos
        parts.append(blocks[firsts[k]:firsts[k + 1]])
        pos += firsts[k + 1] - firsts[k]
    return np.ascontiguousarray(np.concatenate(parts)), t


def run_pictures(lib, mem, decs, block_pad=0, gap=0):
    """ff_prores_decode_pictures_cuda over every picture of the decoded streams in one call: (rc, each stream's frame buffer after it).
    gap > 0: the slices' blocks lie `gap` blocks apart in the coefficient buffer (the table is not the packed one)"""
    works, bufs = [], []
    for d in decs:
        fb = mem.put(d.frame.buf)
        bufs.append(fb)
        laid = [(picture_blocks(d.rec, k), slice_table(d.rec, k)) for k in range(d.rec.n_pics)]
        if gap:
            laid = [spread_slices(b, t, gap, k) for k, (b, t) in enumerate(laid)]
        bl = [mem.put(b, block_pad) for b, _ in laid]
        sl = [mem.put(t) for _, t in laid]
        ws = picture_works(d.frame, d.rec, fb, lambda k: bl[k], lambda k: sl[k])
        for w, (b, _) in zip(ws, laid):
            w.n_blocks = len(b)
        works += ws
    arr = (tables.FFProresPictureWork * max(len(works), 1))(*works)
    rc = lib.ff_prores_decode_pictures_cuda(arr, len(works), None)
    mem.sync()
    return rc, [mem.get(fb, np.uint8, d.frame.buf.shape) for fb, d in zip(bufs, decs)]


def check_frame(d, got):
    """y / u / v equal the reference decoder's byte for byte (padding included); the alpha plane is the pre-filled pattern"""
    for p in range(3):
        a, b = d.frame.plane(got, p), d.frame.plane(d.want, p)
        assert np.array_equal(a, b), (d.spec, "plane", p, np.flatnonzero(a != b)[:8])
    assert np.array_equal(d.frame.plane(got, 3), d.frame.plane(d.frame.buf, 3)), (d.spec, "alpha plane touched")
    rest = np.ones(len(got), bool)
    for p in range(4):
        rest[d.frame.off[p]:d.frame.off[p] + d.frame.ls[p] * d.frame.H] = False
    assert np.array_equal(got[rest], d.frame.buf[rest]), (d.spec, "bytes between planes touched")
