"""TEST INFRASTRUCTURE.  VC-3 / DNxHD encoder cases for tests/test_dnxhd_enc_cpu.py, tests/test_gpu_dnxhd_enc.py and tools/dnxhd_enc_bench.py:
seeded source frames, the options of each case, the product's call (host-compiled or on the GPU) and the reference encoder
(oracle/_ref/libdnxhdencref.so), and a packet parser that reads each macroblock's qscale back from a packet."""
import ctypes as C

import numpy as np

from libav_b200 import tables

vp, i32 = C.c_void_p, C.c_int
FASTINT, FAAN, RD = 1, 6, 2
EINVAL = -22
CIDS = (1235, 1237, 1238, 1241, 1242, 1243, 1250, 1251, 1252, 1253, 1256, 1258, 1259, 1260)
INTERLACED = (1241, 1242, 1243, 1260)
TEN_BIT = (1235, 1241, 1250, 1256)
GEOM = {1235: (1920, 1080), 1237: (1920, 1080), 1238: (1920, 1080), 1241: (1920, 1080), 1242: (1920, 1080), 1243: (1920, 1080),
        1250: (1280, 720), 1251: (1280, 720), 1252: (1280, 720), 1253: (1920, 1080), 1256: (1920, 1080), 1258: (960, 720),
        1259: (1440, 1080), 1260: (1440, 1080)}


class Opts(C.Structure):        # oracle/refbuild/refapi_dnxhd_enc.c RefDnxhdOpts
    _fields_ = [("cid", C.c_int32), ("interlaced", C.c_int32), ("dct_algo", C.c_int32), ("mb_decision", C.c_int32), ("qmax", C.c_int32),
                ("nitris_compat", C.c_int32), ("ibias", C.c_int32)]


def ref():
    """the reference encoder library with prototypes, or None when oracle/_ref was not built"""
    from oracle import loader
    lib = loader.ref_lib("dnxhdenc")
    if lib is None:
        return None
    lib.ref_dnxhd_encode_seq.restype, lib.ref_dnxhd_encode_seq.argtypes = i32, [C.POINTER(Opts), i32, vp, vp, vp, vp]
    lib.ref_dnxhd_cid_entry.restype, lib.ref_dnxhd_cid_entry.argtypes = vp, [i32]
    lib.ref_dnxhd_vlc.restype, lib.ref_dnxhd_vlc.argtypes = i32, [C.POINTER(Opts), vp, vp, vp, vp]
    lib.ref_dnxhd_cid_layout.restype, lib.ref_dnxhd_cid_layout.argtypes = i32, [vp]
    lib.ref_dnxhd_encode_frames.restype, lib.ref_dnxhd_encode_frames.argtypes = i32, [C.POINTER(Opts), i32, vp, vp, vp, vp, i32]
    return lib


def P(a, off=0):
    return C.c_void_p(a.ctypes.data + off)


def frame(cid, content, seed, pad=0, odd=False, tail=None):
    """the three planes of one frame as byte arrays laid out at their linesizes: (planes, linesizes).  Samples are uint8 (8 bit) or
    little-endian uint16 in 0..1023; 10-bit luma planes of 1080-line CIDs carry 8 more lines (1088), filled from `tail` (a seed) or
    replicating the last line.  content: 'natural' (gradients, edges and texture), 'noise', 'flat', 'checker' (0 / max 8 x 8 squares),
    'gradient', 'fields' (natural on even lines, noise on odd ones: one field far harder than the other)"""
    w, h = GEOM[cid]
    ten = cid in TEN_BIT
    mx = 1023 if ten else 255
    r = np.random.default_rng(seed)
    planes, lss = [], []
    for p, pw in enumerate((w, w // 2, w // 2)):
        y, x = np.mgrid[0:h, 0:pw]
        if content == "noise":
            a = r.integers(0, mx + 1, (h, pw))
        elif content == "flat":
            a = np.full((h, pw), int(r.integers(0, mx + 1)))
        elif content == "checker":
            a = (((y >> 3) + (x >> 3) + p) & 1) * mx
        elif content == "gradient":
            a = (x * mx) // max(pw - 1, 1) if p != 1 else (y * mx) // max(h - 1, 1)
        elif content in ("natural", "fields"):
            f = mx / 255.0
            a = (128 + 60 * np.sin(x / (17.0 + 5 * p) + seed) * np.cos(y / 23.0) + 40 * ((x // 37 + y // 29) & 1)) * f
            a = a + r.normal(0, 6 * f, (h, pw))
            if content == "fields":
                a = np.where(y & 1, r.integers(0, mx + 1, (h, pw)), a)
        else:
            raise ValueError(content)
        a = np.clip(np.asarray(a), 0, mx).astype(np.uint16 if ten else np.uint8)
        rows = h + (8 if ten and h == 1080 and p == 0 else 0)
        if rows > h:
            extra = np.random.default_rng(tail).integers(0, 1 << 16, (8, pw)) if tail is not None else np.repeat(a[-1:], 8, 0)
            a = np.concatenate([a, extra.astype(np.uint16)])
        bpp = 2 if ten else 1
        ls = pw * bpp + pad + (1 if odd and not ten else 0)
        buf = np.full((rows, ls), 0x5A, np.uint8)
        buf[:, :pw * bpp] = a.view(np.uint8).reshape(rows, -1)
        planes.append(buf)
        lss.append(ls)
    return planes, lss


class Case:
    """frames encoded in order through one rate-control state"""

    def __init__(self, cid, contents, interlaced=None, dct_algo=0, mb_decision=0, qmax=31, nitris=0, ibias=999999, seed=1, pad=0,
                 odd=False, tails=None):
        self.cid, self.contents, self.dct_algo, self.mb_decision, self.qmax, self.nitris, self.ibias = \
            cid, list(contents), dct_algo, mb_decision, qmax, nitris, ibias
        self.interlaced = (1 if cid in INTERLACED else 0) if interlaced is None else interlaced
        self.seed, self.pad, self.odd = seed, pad, odd
        self.tails = tails or [None] * len(self.contents)
        self.frames = [frame(cid, c, seed + k, pad, odd, t) for k, (c, t) in enumerate(zip(self.contents, self.tails))]

    def __repr__(self):
        return "Case(cid=%d il=%d dct=%d mbd=%d qmax=%d nitris=%d %s seed=%d pad=%d odd=%s)" % (
            self.cid, self.interlaced, self.dct_algo, self.mb_decision, self.qmax, self.nitris, "/".join(self.contents), self.seed,
            self.pad, self.odd)

    def opts(self):
        return Opts(cid=self.cid, interlaced=self.interlaced, dct_algo=self.dct_algo, mb_decision=self.mb_decision, qmax=self.qmax,
                    nitris_compat=self.nitris, ibias=self.ibias)


def ref_encode(lib, case):
    """the reference's packets (None for a failed frame) and (ret, qscale, lambda, quality) after each frame"""
    n = len(case.frames)
    planes = (C.c_void_p * (3 * n))(*[p.ctypes.data for f, _ in case.frames for p in f])
    lss = (C.c_int * (3 * n))(*[ls for _, l in case.frames for ls in l])
    size = lib.ref_dnxhd_cid_entry(case.cid) and C.cast(lib.ref_dnxhd_cid_entry(case.cid), C.POINTER(tables.FFDnxhdCidEntry))[0].frame_size
    out = np.zeros(n * size, np.uint8)
    rc = np.zeros(4 * n, np.int32)
    got = lib.ref_dnxhd_encode_seq(C.byref(case.opts()), n, planes, lss, P(out), P(rc))
    assert got == size, ("reference encode_init failed", case)
    rc = rc.reshape(n, 4)
    return [out[k * size:(k + 1) * size].copy() if rc[k, 0] >= 0 else None for k in range(n)], rc


def run(lib, eref, mem, cases, states=None, cap_delta=0, ws_delta=0, stream=None):
    """ff_dnxhd_encode_frames_cuda over every frame of the cases in one call, each case's frames through its own state (or the states
    given: one index per case).  Returns (rc, packets or None per frame, out_info per frame, states after, raw buffers)"""
    works, infos, outs, st_ptrs = [], [], [], {}
    for ci, c in enumerate(cases):
        key = ci if states is None else states[ci]
        if key not in st_ptrs:
            st_ptrs[key] = mem.put(np.array([1, 2 << 10], np.uint32))
        entry = eref.ref_dnxhd_cid_entry(c.cid)
        size = C.cast(entry, C.POINTER(tables.FFDnxhdCidEntry))[0].frame_size
        for planes, lss in c.frames:
            w = tables.FFDnxhdEncodeWork()
            for p in range(3):
                w.data[p] = mem.put(planes[p])
                w.linesize[p] = lss[p]
            w.cid_table = entry
            w.interlaced, w.dct_algo, w.mb_decision, w.qmax, w.nitris_compat = c.interlaced, c.dct_algo, c.mb_decision, c.qmax, c.nitris
            w.state = st_ptrs[key]
            o = mem.put(np.full(size + 64, 0xCD, np.uint8))
            z = mem.put(np.zeros(2, np.int32))
            w.out, w.out_capacity, w.out_info = o, size + cap_delta, z
            works.append(w); outs.append((o, size)); infos.append(z)
    arr = (tables.FFDnxhdEncodeWork * len(works))(*works)
    need = lib.ff_dnxhd_encode_workspace_cuda(arr, len(works))
    ws = mem.put(np.zeros(max(need, 1), np.uint8))
    rc = lib.ff_dnxhd_encode_frames_cuda(arr, len(works), C.c_void_p(ws), need + ws_delta, stream)
    if rc:
        return rc, None, None, None, None
    mem.sync()
    info = [mem.get(z, np.int32, (2,)).copy() for z in infos]
    raws = [mem.get(o, np.uint8, (size + 64,)).copy() for o, size in outs]
    pkts = [r[:size].copy() if i[0] > 0 else None for r, (o, size), i in zip(raws, outs, info)]
    sts = {k: mem.get(p, np.uint32, (2,)).copy() for k, p in st_ptrs.items()}
    return rc, pkts, info, sts, raws


def mb_qscales(pkt, cid):
    """the qscale of each slice's first macroblock, read from the packet: a slice starts at its MSIP offset with that macroblock's 12-bit
    field (the later macroblocks' positions need the VLC tables)"""
    w, h = GEOM[cid]
    nf = 2 if cid in INTERLACED else 1
    cu = len(pkt) // nf
    out = []
    for f in range(nf):
        b = pkt[f * cu:(f + 1) * cu]
        ns = int(b[0x16d])
        for y in range(ns):
            off = 640 + int.from_bytes(bytes(b[0x170 + 4 * y:0x174 + 4 * y]), "big")
            out.append((int(b[off]) << 4 | int(b[off + 1]) >> 4) >> 1)
    return out


def compare(case, k, got, want):
    """byte-identical packets; on a difference the first row whose first macroblock's qscale differs, or the first differing byte"""
    if (got is None and want is None) or (got is not None and want is not None and np.array_equal(got, want)):
        return
    msg = [repr(case), "frame %d" % k, "got %s, want %s" % ("no packet" if got is None else "a packet", "no packet" if want is None else "a packet")]
    if got is not None and want is not None:
        qa, qb = mb_qscales(got, case.cid), mb_qscales(want, case.cid)
        bad = [i for i, (a, b) in enumerate(zip(qa, qb)) if a != b]
        if bad:
            msg.append("first slice whose first macroblock has another qscale: %d (%d vs %d)" % (bad[0], qa[bad[0]], qb[bad[0]]))
        d = np.flatnonzero(got != want)
        msg.append("first differing byte: %d" % d[0])
    raise AssertionError("; ".join(msg))


def check_states(lib, eref, mem, case):
    """the case's frames one call each through one state: the state after every frame equals the reference context's qscale / lambda"""
    _, wrc = ref_encode(eref, case)
    st = mem.put(np.array([1, 2 << 10], np.uint32))
    for f in range(len(case.frames)):
        one = Case.__new__(Case)
        one.__dict__.update(case.__dict__)
        one.frames = [case.frames[f]]
        works = run_frames(eref, mem, one, st)
        arr = (tables.FFDnxhdEncodeWork * 1)(*works)
        need = lib.ff_dnxhd_encode_workspace_cuda(arr, 1)
        ws = mem.put(np.zeros(need, np.uint8))
        assert lib.ff_dnxhd_encode_frames_cuda(arr, 1, C.c_void_p(ws), need, None) == 0, lib.avb200_last_error()
        mem.sync()
        assert list(mem.get(st, np.uint32, (2,))) == [wrc[f, 1], wrc[f, 2]], (case, f, list(mem.get(st, np.uint32, (2,))), wrc[f])


def run_frames(eref, mem, case, state):
    """the works of a case's frames through one state pointer"""
    entry = eref.ref_dnxhd_cid_entry(case.cid)
    size = C.cast(entry, C.POINTER(tables.FFDnxhdCidEntry))[0].frame_size
    works = []
    for planes, lss in case.frames:
        w = tables.FFDnxhdEncodeWork()
        for p in range(3):
            w.data[p] = mem.put(planes[p])
            w.linesize[p] = lss[p]
        w.cid_table = entry
        w.interlaced, w.dct_algo, w.mb_decision, w.qmax, w.nitris_compat = case.interlaced, case.dct_algo, case.mb_decision, case.qmax, case.nitris
        w.state, w.out, w.out_capacity, w.out_info = state, mem.put(np.zeros(size, np.uint8)), size, mem.put(np.zeros(2, np.int32))
        works.append(w)
    return works


def check(lib, eref, mem, cases, states=None):
    """every frame of the cases in one call against the reference: packets, out_info and the state after the last frame of each state"""
    rc, pkts, info, sts, raws = run(lib, eref, mem, cases, states)
    assert rc == 0, lib.avb200_last_error()
    k = 0
    for ci, c in enumerate(cases):
        want, wrc = ref_encode(eref, c)
        for f in range(len(c.frames)):
            compare(c, f, pkts[k], want[f])
            assert info[k][0] == (EINVAL if wrc[f, 0] < 0 else len(want[f])), (c, f, info[k], wrc[f])
            assert info[k][1] == wrc[f, 1] * 118, (c, f, info[k], wrc[f])
            size = len(raws[k]) - 64
            assert (raws[k][size:] == 0xCD).all(), (c, f, "wrote past frame_size")
            k += 1
        if states is None:
            assert list(sts[ci]) == [wrc[-1, 1], wrc[-1, 2]], (c, "state", list(sts[ci]), wrc[-1])
    return pkts, info
