"""TEST INFRASTRUCTURE.  ProRes decoder cases for tests/test_prores_dec_cpu.py, tests/test_gpu_prores_dec.py and tools/prores_dec_bench.py:
the reference decoder with the checked reader (oracle/_ref/libproresdecref.so), packets from the reference encoder
(oracle/_ref/libproresencref.so), a packet parser and the header edits built on it, and the product's call (host-compiled or on the GPU)
compared with the reference byte for byte, the sentinel in what the decoder does not write and the alpha plane included."""
import ctypes as C

import numpy as np

import prores_enc_util as E
from libav_b200 import tables

vp, i32 = C.c_void_p, C.c_int
SENTINEL = 0xA5
INVALIDDATA = -0x3ebbb1b7
NINFO = 13


def ref():
    """the reference decoder library with prototypes, or None when oracle/_ref was not built"""
    from oracle import loader
    lib = loader.ref_lib("proresdec")
    if lib is None:
        return None
    lib.ref_prores_dec_decode.restype, lib.ref_prores_dec_decode.argtypes = None, [vp, vp, i32, i32, i32, vp, vp, vp]
    lib.ref_prores_dec_tables.restype, lib.ref_prores_dec_tables.argtypes = i32, [vp]
    lib.ref_prores_dec_pix_fmts.restype, lib.ref_prores_dec_pix_fmts.argtypes = None, [vp]
    lib.ref_prores_dec_neg_usr32.restype, lib.ref_prores_dec_neg_usr32.argtypes = C.c_uint32, [C.c_uint32, i32]
    lib.ref_prores_dec_decode_frames.restype = i32
    lib.ref_prores_dec_decode_frames.argtypes = [vp, vp, i32, i32, i32, vp, vp, i32]
    return lib


class Pkt:
    """a packet and the dimensions it is decoded at"""

    def __init__(self, data, w, h, name=""):
        self.data, self.w, self.h, self.name = bytes(data), w, h, name

    def __repr__(self):
        return "Pkt(%s %dx%d, %d bytes)" % (self.name, self.w, self.h, len(self.data))


# ------------------------------------------------------------------------------------------------------------------------ real packets
def encode(eref, fmt, w, h, interlaced=0, profile=2, mbs_per_slice=8, alpha_bits=16, content="natural", seed=1, **kw):
    c = E.Case(fmt, w, h, interlaced=interlaced, profile=profile, mbs_per_slice=mbs_per_slice, alpha_bits=alpha_bits, content=content,
               seed=seed, **kw)
    pkt, _ = E.ref_encode(eref, c)
    return Pkt(pkt, w, h, "enc(fmt=%d il=%d prof=%d mps=%d ab=%d %dx%d)" % (fmt, interlaced, profile, mbs_per_slice, alpha_bits, w, h))


# ------------------------------------------------------------------------------------------------------------------------------ parser
def rb16(b, o):
    return b[o] << 8 | b[o + 1]


def rb32(b, o):
    return b[o] << 24 | b[o + 1] << 16 | b[o + 2] << 8 | b[o + 3]


def parse(pkt):
    """{'hdr': frame header size, 'pics': [{'at', 'hdr', 'size', 'n', 'index', 'slices': [(offset, size)]}]} of a well-formed packet"""
    b = pkt.data
    hdr = rb16(b, 8)
    il = (b[20] >> 2) & 3
    at = 8 + hdr
    pics = []
    for _ in range(2 if il else 1):
        ph = b[at] >> 3
        n = rb16(b, at + 5)
        idx = at + ph
        off = idx + 2 * n
        sl = []
        for s in range(n):
            sz = rb16(b, idx + 2 * s)
            sl.append((off, sz))
            off += sz
        pics.append(dict(at=at, hdr=ph, size=rb32(b, at + 1), n=n, index=idx, slices=sl))
        at += rb32(b, at + 1)
    return dict(hdr=hdr, pics=pics)


def edit(pkt, name, fn):
    b = bytearray(pkt.data)
    out = fn(b, parse(pkt))
    b = out if isinstance(out, bytearray) else b
    return Pkt(b, pkt.w, pkt.h, pkt.name + "+" + name)


def set16(b, o, v):
    b[o:o + 2] = (v & 0xffff).to_bytes(2, "big")


def set32(b, o, v):
    b[o:o + 4] = (v & 0xffffffff).to_bytes(4, "big")


def plane_span(b, s, p):
    """(first byte, size) of plane p (0 Y, 1 U, 2 V) of the slice at (offset, size), as decode_slice reads its header"""
    off, size = s
    hdr = b[off] >> 3
    ys, us = rb16(b, off + 2), rb16(b, off + 4)
    vs = rb16(b, off + 6) if hdr > 7 else size - hdr - ys - us
    starts = [off + hdr, off + hdr + ys, off + hdr + ys + us]
    return starts[p], (ys, us, vs)[p]


def zero_dc_run(b, s, p, lead, size=None):
    """plane p of slice s filled with zeros except one 1 bit after `lead` zero bits: FIRST_DC_CB's exp-Golomb length is then
    2 lead + 6 (up to 68), and the shift count 32 - len goes negative for lead > 13.  size: first set the Y (p 0) or U (p 1) plane's size
    to this many bytes, so that DC decoding runs to the clamp position and AC decoding ends there without an error: the plane is written"""
    if size is not None:
        set16(b, s[0] + 2 + 2 * p, size)
    start, size = plane_span(b, s, p)
    for k in range(size):
        b[start + k] = 0
    if lead // 8 < size:
        b[start + lead // 8] = 0x80 >> (lead % 8)


# ----------------------------------------------------------------------------------------------------------------------------- decoding
def probe(lib, pkt):
    info = tables.FFProresFrameInfo()
    buf = np.frombuffer(pkt.data, np.uint8).copy()
    ret = lib.ff_prores_probe_cuda(buf.ctypes.data, len(buf), pkt.w, pkt.h, C.byref(info))
    return ret, info


def tables_pix_fmts():
    return (66, 70, 92, 94)            # FF_PRORES_PIX_FMT_* (tests check them against the reference build)


def ref_decode(dref, pkts, lines_of, pad=0):
    """packets through ONE reference context in turn (a list of one: a fresh context): ([planes per packet], [info rows])"""
    n = len(pkts)
    bufs = [np.frombuffer(p.data, np.uint8).copy() for p in pkts]
    ptrs = (C.c_void_p * n)(*[b.ctypes.data for b in bufs])
    sizes = (C.c_int * n)(*[len(b) for b in bufs])
    allp, ptr4, ls4 = [], [], []
    for k, p in enumerate(pkts):
        mbw = (p.w + 15) // 16
        lss = [32 * mbw + pad] * 4                                     # wide enough for any format the header may announce
        planes = [np.full((lines_of[k], ls), SENTINEL, np.uint8) for ls in lss]
        allp.append(planes)
        ptr4 += [pl.ctypes.data for pl in planes]
        ls4 += lss
    info = np.zeros(NINFO * n, np.int32)
    w, h = pkts[0].w, pkts[0].h
    assert all((p.w, p.h) == (w, h) for p in pkts)
    dref.ref_prores_dec_decode(ptrs, sizes, n, w, h, (C.c_void_p * (4 * n))(*ptr4), (C.c_int * (4 * n))(*ls4), info.ctypes.data)
    return allp, info.reshape(n, NINFO)


def run(lib, mem, pkts, pad=0, ws_delta=0, ws_offset=0, mutate=None, stream=None, dev_pkts=None):
    """ff_prores_decode_frames_cuda over the packets in one call: (rc, [planes per packet], [info per packet])"""
    works, outs, infos, keep = [], [], [], []
    for k, pkt in enumerate(pkts):
        ret, info = probe(lib, pkt)
        assert ret == 0, (pkt, ret)
        mbw = (pkt.w + 15) // 16
        lss = [32 * mbw + pad] * 4
        planes = [np.full((info.lines, ls), SENTINEL, np.uint8) for ls in lss]
        w = tables.FFProresDecodeWork()
        hb = np.frombuffer(pkt.data, np.uint8).copy()
        keep.append(hb)
        w.pkt_host, w.size, w.width, w.height = hb.ctypes.data, len(hb), pkt.w, pkt.h
        w.pkt = dev_pkts[k] if dev_pkts is not None else mem.put(hb)
        ptrs = []
        for p in range(4):
            ptrs.append(mem.put(planes[p]))
            w.data[p], w.linesize[p], w.lines[p] = ptrs[-1], lss[p], info.lines
        if mutate:
            mutate(w)
        works.append(w); outs.append((ptrs, planes)); infos.append(info)
    arr = (tables.FFProresDecodeWork * len(works))(*works)
    need = lib.ff_prores_decode_workspace_cuda(arr, len(works))
    ws = mem.put(np.zeros(max(need, 1) + ws_offset, np.uint8))
    rc = lib.ff_prores_decode_frames_cuda(arr, len(works), C.c_void_p(ws + ws_offset), need + ws_delta, stream)
    if rc:
        return rc, None, infos
    mem.sync()
    res = [[mem.get(p, np.uint8, pl.shape) for p, pl in zip(ptrs, planes)] for ptrs, planes in outs]
    return rc, res, infos


def check_probe(lib, dref, pkt, guard=16):
    """the probe against the reference's decode_frame: its return value before get_buffer, or the frame info.  Returns the info when the
    probe accepted the packet, else None."""
    ret, info = probe(lib, pkt)
    lines = max(info.lines, 16) + guard if ret == 0 else 64
    _, row = ref_decode(dref, [pkt], [lines])
    row = row[0]
    if ret != 0:
        assert ret == row[0] and row[9] == 0, (pkt, ret, list(row))            # the reference failed before get_buffer
        return None
    fm = np.zeros(4, np.int32)
    dref.ref_prores_dec_pix_fmts(fm.ctypes.data)
    assert row[9] == 1, (pkt, list(row))
    assert info.result == row[0], (pkt, info.result, row[0])
    assert info.pictures == row[8], (pkt, info.pictures, row[8])
    assert fm[list(tables_pix_fmts()).index(info.pix_fmt)] == row[2], (pkt, info.pix_fmt, row[2])
    assert (info.interlaced_frame, info.top_field_first) == (row[3], row[4]), (pkt, list(row))
    assert (info.color_primaries, info.color_trc, info.colorspace) == (row[5], row[6], row[7]), (pkt, list(row))
    if info.pictures:
        assert info.lines == (row[12] * 16) << info.interlaced_frame, (pkt, info.lines, row[12])
    return info


def check(lib, dref, mem, pkts, pad=0, stream=None, dev_pkts=None):
    """decode the packets in one call and compare every plane and the info with the reference, one fresh context per packet"""
    for p in {(p.data, p.w, p.h): p for p in pkts}.values():
        assert check_probe(lib, dref, p) is not None, p
    rc, res, infos = run(lib, mem, pkts, pad=pad, stream=stream, dev_pkts=dev_pkts)
    assert rc == 0, lib.avb200_last_error()
    wants = {}
    for k, (pkt, got, info) in enumerate(zip(pkts, res, infos)):
        key = (pkt.data, pkt.w, pkt.h)
        if key not in wants:
            wants[key] = ref_decode(dref, [pkt], [info.lines + 16], pad=pad)[0][0]
        want = wants[key]
        alpha = info.pix_fmt in tables_pix_fmts()[2:]
        for p in range(4):
            assert (want[p][info.lines:] == SENTINEL).all(), ("reference wrote past info.lines", pkt, p)
            a, b = got[p], want[p][:info.lines]
            if p == 3 and not alpha:
                assert (b == SENTINEL).all() and (a == SENTINEL).all(), pkt
            if not np.array_equal(a, b):
                bad = np.argwhere(a != b)
                raise AssertionError("%r plane %d differs at %d places, first (line, byte) %s: got %d want %d" % (
                    pkt, p, len(bad), tuple(bad[0]), a[tuple(bad[0])], b[tuple(bad[0])]))
    return infos
