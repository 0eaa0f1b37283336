"""TEST INFRASTRUCTURE.  VC-3 / DNxHD decoder cases for tests/test_dnxhd_dec_cpu.py, tests/test_gpu_dnxhd_dec.py and tools/dnxhd_dec_bench.py:
the reference decoder (oracle/_ref/libdnxhddecref.so) and its CID table, real packets from the reference encoder
(oracle/_ref/libdnxhdencref.so), a packet synthesiser that writes headers, scan indices and random symbol streams from the exported CID
entries (the encoder never writes 4:4:4 or mbaff), and the product's call (host-compiled or on the GPU) compared byte for byte with the
reference, sentinel included."""
import ctypes as C

import numpy as np

import dnxhd_enc_util as E
from libav_b200 import tables

vp, i32 = C.c_void_p, C.c_int
SENTINEL = 0xA5
INVALIDDATA, ENOSYS, EINVAL = -0x3ebbb1b7, -38, -22


def ref():
    """the reference decoder library with prototypes, or None when oracle/_ref was not built"""
    from oracle import loader
    lib = loader.ref_lib("dnxhddec")
    if lib is None:
        return None
    lib.ref_dnxhd_decode.restype, lib.ref_dnxhd_decode.argtypes = i32, [vp, i32, i32, vp, vp, i32, vp, vp]
    lib.ref_dnxhd_cid_table.restype, lib.ref_dnxhd_cid_table.argtypes = vp, [vp]
    lib.ref_dnxhd_pix_fmts.restype, lib.ref_dnxhd_pix_fmts.argtypes = None, [vp]
    lib.ref_dnxhd_decode_frames.restype, lib.ref_dnxhd_decode_frames.argtypes = i32, [vp, vp, i32, vp, vp, i32, i32]
    return lib


def cid_table(dref):
    """(pointer to the reference's ff_dnxhd_cid_table, its length, {cid: FFDnxhdCidEntry})"""
    n = C.c_int()
    p = dref.ref_dnxhd_cid_table(C.byref(n))
    arr = C.cast(p, C.POINTER(tables.FFDnxhdCidEntry))
    return C.c_void_p(p), n.value, {arr[k].cid: arr[k] for k in range(n.value)}


def u8(ptr, n):
    return np.ctypeslib.as_array(C.cast(ptr, C.POINTER(C.c_uint8)), (n,)).copy()


def u16(ptr, n):
    return np.ctypeslib.as_array(C.cast(ptr, C.POINTER(C.c_uint16)), (n,)).copy()


def codes(e):
    """the entry's code tables as Python lists"""
    ndc = e.bit_depth + 4
    return dict(ac_codes=u16(e.ac_codes, 257), ac_bits=u8(e.ac_bits, 257), ac_level=u8(e.ac_level, 257),
                ac_index=u8(e.ac_index_flag, 257), ac_run=u8(e.ac_run_flag, 257), run_codes=u16(e.run_codes, 62),
                run_bits=u8(e.run_bits, 62), run=u8(e.run, 62), dc_codes=u8(e.dc_codes, ndc), dc_bits=u8(e.dc_bits, ndc))


# ------------------------------------------------------------------------------------------------------------------------ real packets
def real_packets(eref, cid, contents, interlaced=None, mb_decision=0, seed=1):
    """the reference encoder's packets for frames of the given contents; a frame the rate control cannot fit even at qmax 69 (noise at
    the lower bit rates) is encoded from natural content instead"""
    out = []
    for k, c in enumerate(contents):
        for content in (c, "natural"):
            pk, _ = E.ref_encode(eref, E.Case(cid, [content], interlaced=interlaced, mb_decision=mb_decision, qmax=69, seed=seed + k))
            if pk[0] is not None:
                break
        assert pk[0] is not None
        out.append(bytes(pk[0]))
    return out


# ------------------------------------------------------------------------------------------------------------------------- synthesiser
class Bits:
    def __init__(self):
        self.v, self.n = 0, 0

    def put(self, code, n):
        n = int(n)
        if n:
            self.v = (self.v << n) | (int(code) & ((1 << n) - 1))
            self.n += n

    def bytes(self):
        pad = (-self.n) % 8
        return ((self.v << pad).to_bytes((self.n + pad) // 8, "big") if self.n else b"")


class Synth:
    """options of a synthesised packet.  qscales: the values qscale is drawn from; eob: the chance of an EOB after each coefficient;
    big: the chance that a coefficient takes the largest level and index bits; runs: the chance of drawing a run code (the runs then push
    i past 63 now and then); dc_big: the chance of the longest DC difference, always positive (DC drift); mbaff / ilmb: the mbaff flag and
    the chance of interlaced_mb; is444: the 4:4:4 prefix; header_width / mb_height / heights: header fields; tail: bytes after the last
    row; scan: 'inorder', 'shuffle' (rows stored out of order), 'overlap' (every row at the same offset), 'end' (the last row's index
    at the packet's end) or 'cu_end' (the first field's last row two bytes before the second field); weights: (luma, chroma) weights of
    the entry the packet is decoded with -- then the synthesiser never pushes a block past coefficient 63 and leaves in .expected the
    dequantised coefficients of the first unit's rows, [row][mb][block][64], and in .wraps how many products reached 2^31"""

    def __init__(self, cid, seed=1, qscales=(1, 2, 4, 8, 16, 31), eob=0.25, big=0.0, runs=0.3, dc_big=0.0, mbaff=False, ilmb=0.0,
                 is444=False, header_width=None, mb_height=None, scan="inorder", fields=(0, 1), bits=None, pad=64, weights=None):
        self.__dict__.update(locals())
        del self.__dict__["self"]


def synth(dref, s):
    """one packet of CID s.cid built by the options in s"""
    _, _, entries = cid_table(dref)
    e = entries[s.cid]
    T = codes(e)
    r = np.random.default_rng(s.seed)
    bd = e.bit_depth if s.bits is None else s.bits
    nu = 2 if e.interlaced else 1
    mbw = e.width // 16
    mbh_full = (e.height + 15) // 16 // nu
    mbh = mbh_full if s.mb_height is None else s.mb_height
    nblk = 12 if s.is444 and bd == 10 else 8
    ac_ok = [k for k in range(257) if T["ac_bits"][k]]
    eobs = [k for k in ac_ok if T["ac_level"][k] == 0]
    nonz = [k for k in ac_ok if T["ac_level"][k] != 0]
    big_k = max(nonz, key=lambda k: (T["ac_index"][k], T["ac_level"][k]))
    ib = 4 if bd == 8 else 6
    bias, shift = (32, 6) if bd == 8 or nblk == 12 else (8, 4)
    model = None
    if s.weights is not None:                                         # the expected coefficients of the first unit's rows
        model = np.zeros((mbh, mbw, nblk, 64), np.int16)
        s.wraps = 0
    units = []
    for u in range(nu):
        rows = []
        for y in range(mbh):
            b = Bits()
            last_dc = [1 << (bd + 2)] * 3
            for x in range(mbw):
                q = int(r.choice(s.qscales))
                if s.mbaff:
                    b.put(int(r.random() < s.ilmb), 1)
                    b.put(q & 1023, 10)
                else:
                    b.put(q & 2047, 11)
                b.put(0, 1)
                q = q & 1023 if s.mbaff else q & 2047
                for n in range(nblk):
                    comp = (n >> 1) % 3 if nblk == 12 else (1 + (n & 1) if n & 2 else 0)
                    ndc = len(T["dc_bits"])
                    d = ndc - 1 if r.random() < s.dc_big else int(r.integers(0, ndc))
                    b.put(T["dc_codes"][d], T["dc_bits"][d])
                    if d:
                        dv = ((1 << d) - 1) if s.dc_big and r.random() < s.dc_big else int(r.integers(0, 1 << d))
                        b.put(dv, d)
                        if model is not None:
                            last_dc[comp] += dv if dv >> (d - 1) else dv - ((1 << d) - 1)
                    if model is not None and u == 0:
                        blk = model[y, x, n]
                        blk[0] = int16(last_dc[comp])
                    i = 1
                    for _ in range(64):
                        if r.random() < s.eob:
                            break
                        k = big_k if r.random() < s.big else int(r.choice(nonz))
                        sg = int(r.integers(0, 2))
                        iv = None
                        if T["ac_index"][k]:
                            iv = (1 << ib) - 1 if k == big_k and s.big else int(r.integers(0, 1 << ib))
                        j = None
                        if T["ac_run"][k]:
                            j = int(r.integers(0, 62)) if r.random() < s.runs else int(np.argmin(T["run"]))
                        pos = i + (int(T["run"][j]) if j is not None else 0)
                        if model is not None and pos > 63:                    # the model stays clear of the damaged-block break
                            break
                        b.put(T["ac_codes"][k], T["ac_bits"][k])
                        b.put(sg, 1)
                        if iv is not None:
                            b.put(iv, ib)
                        if j is not None:
                            b.put(T["run_codes"][j], T["run_bits"][j])
                        if model is not None and u == 0:
                            level = int(T["ac_level"][k]) + ((iv or 0) << 6)
                            w = int(s.weights[1 if comp else 0][pos])
                            wrapped = (2 * level + 1) * q * w
                            s.wraps += wrapped >= 1 << 31
                            blk[ZIGZAG[pos]] = dequant(level, sg, q, w, bias, shift)
                        i = pos + 1
                    k = int(r.choice(eobs))
                    b.put(T["ac_codes"][k], T["ac_bits"][k])
            rows.append(b.bytes() + b"\0" * ((-len(b.bytes())) % 4))
        order = list(range(mbh))
        if s.scan == "shuffle":
            r.shuffle(order)
        data, offs = b"", [0] * mbh
        for y in order:
            offs[y] = len(data)
            data += rows[y]
        if s.scan == "overlap":
            offs = [0] * mbh
        hdr = bytearray(0x280)
        hdr[0:5] = bytes([0, 0, 2, 0x80, 2 if s.is444 else 1])
        hdr[5] = (2 | (s.fields[u] & 1)) if e.interlaced else 1
        hdr[6] = 0x80 | (32 if s.mbaff else 0)
        hdr[7] = 0xa0
        hh = e.height >> (nu - 1)
        hdr[0x18:0x1a] = hh.to_bytes(2, "big")
        hdr[0x1a:0x1c] = (e.width if s.header_width is None else s.header_width).to_bytes(2, "big")
        hdr[0x21] = 0x58 if bd == 10 else 0x38
        hdr[0x28:0x2c] = s.cid.to_bytes(4, "big")
        hdr[0x16d] = mbh
        body = data + b"\0" * s.pad
        if s.scan == "end":                                           # the last row reads nothing but the zero bits past the packet
            body += b"\0" * (e.coding_unit_size - 0x280 - len(body))
            offs[mbh - 1] = len(body)
        if s.scan == "cu_end" and u == 0:                             # the first field's last row runs into the second field's header
            body += b"\0" * (e.coding_unit_size - 0x280 - len(body))
            offs[mbh - 1] = len(body) - 2
        for y in range(mbh):
            hdr[0x170 + 4 * y:0x174 + 4 * y] = offs[y].to_bytes(4, "big")
        unit = bytes(hdr) + body
        units.append(unit)
    cu = max(e.coding_unit_size, max(len(x) for x in units))
    if nu == 2 and cu > e.coding_unit_size:
        raise ValueError("synthesised field larger than the coding unit")
    out = b""
    for k, unit in enumerate(units):
        out += unit if (k == nu - 1 and s.scan == "end") else unit + b"\0" * (cu - len(unit))
    s.expected = model
    return out


ZIGZAG = [0] * 64                                                     # ff_zigzag_direct
_k = 0
for _s in range(15):
    _r0, _r1 = (0, _s) if _s < 8 else (_s - 7, 7)
    for _n in range(_r1 - _r0 + 1):
        _r = _r0 + _n if _s & 1 else _r1 - _n
        ZIGZAG[_k] = 8 * _r + _s - _r
        _k += 1


def int16(v):
    return ((int(v) + 32768) & 0xffff) - 32768


def dequant(level, sign_bit, qscale, weight, bias, shift):
    """dnxhd_decode_dct_block's coefficient: (2 level + 1) qscale weight in 32-bit two's complement, the bias unless an 8-bit weight equals
    it, an arithmetic shift, the sign, then int16"""
    v = ((2 * level + 1) * qscale * weight) & 0xffffffff
    if bias < 32 or weight != bias:
        v = (v + bias) & 0xffffffff
    lv = (v - (1 << 32) if v >= 1 << 31 else v) >> shift
    sg = -sign_bit
    return int16((lv ^ sg) - sg)


# ---------------------------------------------------------------------------------------------------------------------------- decoding
def info_of(lib, pkt, cids, n):
    info = tables.FFDnxhdFrameInfo()
    ret = lib.ff_dnxhd_probe_cuda(pkt, len(pkt), cids, n, C.byref(info))
    return ret, info


def planes_for(info, pad, lines):
    """sentinel planes (y, u, v) with their linesizes for a frame of this info"""
    bpp = 1 if info.pix_fmt == 4 else 2
    cw = info.width if info.pix_fmt == 70 else info.width // 2
    lss = [info.width * bpp + pad, cw * bpp + pad, cw * bpp + pad]
    return [np.full((lines, ls), SENTINEL, np.uint8) for ls in lss], lss


def ref_decode(dref, pkt, info, gray=0, pad=0, guard=16):
    """the reference's planes (lines + guard lines each), its info row and damaged count"""
    lines = max(info.lines, info.height) + guard                       # get_buffer allocates the frame's height, the decoder writes lines
    planes, lss = planes_for(info, pad, lines)
    arr = (C.c_void_p * 3)(*[p.ctypes.data for p in planes])
    ls = (C.c_int * 3)(*lss)
    out = np.zeros(11, np.int32)
    dmg = C.c_int()
    buf = np.frombuffer(pkt, np.uint8).copy()
    ret = dref.ref_dnxhd_decode(buf.ctypes.data, len(pkt), gray, arr, ls, lines, out.ctypes.data, C.byref(dmg))
    return ret, planes, out, dmg.value


def run(lib, mem, pkts, cids, n_cids, gray=0, pad=0, ws_delta=0, mutate=None):
    """ff_dnxhd_decode_frames_cuda over the packets in one call: (rc, [planes per packet], [info per packet])"""
    works, outs, infos = [], [], []
    keep = []
    for pkt in pkts:
        ret, info = info_of(lib, pkt, cids, n_cids)
        assert ret == 0, ret
        planes, lss = planes_for(info, pad, info.lines)
        w = tables.FFDnxhdDecodeWork()
        hb = np.frombuffer(pkt, np.uint8).copy()
        keep.append(hb)
        w.pkt_host, w.pkt, w.size = hb.ctypes.data, mem.put(hb), len(pkt)
        ptrs = []
        for p in range(3):
            ptrs.append(mem.put(planes[p]))
            w.data[p], w.linesize[p], w.lines[p] = ptrs[-1], lss[p], info.lines
        w.gray = gray
        if mutate:
            mutate(w)
        works.append(w); outs.append((ptrs, planes)); infos.append(info)
    arr = (tables.FFDnxhdDecodeWork * len(works))(*works)
    need = lib.ff_dnxhd_decode_workspace_cuda(arr, len(works), cids, n_cids)
    ws = mem.put(np.zeros(max(need, 1), np.uint8))
    rc = lib.ff_dnxhd_decode_frames_cuda(arr, len(works), cids, n_cids, C.c_void_p(ws), need + ws_delta, None)
    if rc:
        return rc, None, infos
    mem.sync()
    res = [[mem.get(p, np.uint8, pl.shape) for p, pl in zip(ptrs, planes)] for ptrs, planes in outs]
    return rc, res, infos


def check(lib, dref, mem, pkts, gray=0, pad=0):
    """decode the packets in one call and compare every plane and the info with the reference, one fresh context per packet; returns the
    total damaged-block count the reference logged"""
    cids, n, _ = cid_table(dref)
    fmts = np.zeros(3, np.int32)
    dref.ref_dnxhd_pix_fmts(fmts.ctypes.data)
    rc, res, infos = run(lib, mem, pkts, cids, n, gray=gray, pad=pad)
    assert rc == 0, lib.avb200_last_error()
    damaged = 0
    for k, (pkt, got, info) in enumerate(zip(pkts, res, infos)):
        ret, want, row, dmg = ref_decode(dref, pkt, info, gray=gray, pad=pad)
        damaged += dmg
        cu = C.cast(cids, C.POINTER(tables.FFDnxhdCidEntry))[[e.cid for e in C.cast(cids, C.POINTER(tables.FFDnxhdCidEntry))[:n]].index(
            info.cid)].coding_unit_size
        assert ret == len(pkt) - (cu if info.interlaced_frame else 0), (ret, len(pkt))          # dnxhd_decode_frame returns buf_size
        assert row[1] == 1 and row[10] == 1
        assert (row[2], row[3], row[4]) == (info.cid, info.width, info.height)
        assert row[5] == {4: fmts[0], 66: fmts[1], 70: fmts[2]}[info.pix_fmt]
        assert (row[6], row[7], row[8], row[9]) == (info.interlaced_frame, info.top_field_first, info.sar_num, info.sar_den)
        for p in range(3):
            assert (want[p][info.lines:] == SENTINEL).all(), ("reference wrote past info.lines", k, p)
            a, b = got[p], want[p][:info.lines]
            if not np.array_equal(a, b):
                bad = np.argwhere(a != b)
                raise AssertionError("packet %d plane %d differs at %d places, first (line, byte) %s: got %d want %d" % (
                    k, p, len(bad), tuple(bad[0]), a[tuple(bad[0])], b[tuple(bad[0])]))
    return damaged
