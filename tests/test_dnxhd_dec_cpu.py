"""The VC-3 / DNxHD decoder (libav_b200/csrc/dnxhd_dec.cu + dnxhd_dec.cuh) compiled as host C++ (tests/hostsim/dnxhd_dec_hostsim.cpp) against
the reference decoder (oracle/_ref/libdnxhddecref.so: dnxhddec.c, unmodified), one fresh context per packet: every plane byte for byte,
the sentinel in what the decoder does not write included, and the frame info.  Real packets from the reference encoder and synthesised
ones (4:4:4, mbaff, extreme levels and qscales, damaged blocks, DC drift, zero-bit tails, odd scan indices, short mb_height, SAR), the
probe's return codes on malformed headers, and every refusal.

Mutations of dnxhd_dec.cuh this file catches (failed tests of 46): bounding each row's reads at its coding unit instead of the packet 1
(row_reads_second_field); saturating the level instead of wrapping 1 (test_dequantisation_wraps_with_caller_weights: the weights of
ff_dnxhd_cid_table never take the product to 2^31, see test_reachability); resetting last_dc per macroblock 42; ignoring interlaced_mb 4."""
import ctypes as C

import numpy as np
import pytest

import hostsim_build
import prores_util as PU
import dnxhd_enc_util as E
import dnxhd_dec_util as D
from libav_b200 import tables


@pytest.fixture(scope="session")
def dref(built):
    lib, elib = D.ref(), E.ref()
    if lib is None or elib is None:
        pytest.skip("oracle/_ref not built (no reference tree in this environment)")
    return lib


@pytest.fixture(scope="session")
def eref(dref):
    return E.ref()


@pytest.fixture(scope="session")
def hs(built):
    return hostsim_build.load()


def real_groups():
    """every CID the reference encoder writes; both field orders; fast and RD; natural, noise and flat content"""
    g = {}
    for k, cid in enumerate(E.CIDS):
        g["cid%d" % cid] = (cid, ["natural" if k % 3 else "noise"], None, E.RD if k % 2 else 0)
    for cid in E.INTERLACED:
        g["cid%d_bff" % cid] = (cid, ["natural"], 2, 0)
    g["flat_checker"] = (1252, ["flat", "checker"], None, 0)
    return g


REAL = real_groups()

SYNTH = {
    "444": D.Synth(1256, seed=1, mb_height=6, is444=True, eob=0.3),
    "444_prefix_at_8bit": D.Synth(1258, seed=2, is444=True, mb_height=10),
    "mbaff_1260": D.Synth(1260, seed=3, mbaff=True, ilmb=0.5, mb_height=8, qscales=(1, 5, 1023)),
    "mbaff_1252": D.Synth(1252, seed=4, mbaff=True, ilmb=0.5, qscales=(0, 1, 1023)),
    "mbaff_interlaced_1243": D.Synth(1243, seed=5, mbaff=True, ilmb=0.5, mb_height=6),
    "qscale_0_1_2047": D.Synth(1258, seed=6, qscales=(0, 1, 2047)),
    "wrap_8bit": D.Synth(1258, seed=7, qscales=(2047,), big=0.5, eob=0.1),
    "wrap_10bit": D.Synth(1250, seed=8, qscales=(2047,), big=0.5, eob=0.1, mb_height=10),
    "damaged_runs": D.Synth(1252, seed=9, runs=1.0, eob=0.02),
    "dc_drift": D.Synth(1258, seed=10, dc_big=0.9, eob=0.6),
    "dc_drift_10bit": D.Synth(1250, seed=11, dc_big=0.9, eob=0.6, mb_height=12),
    "zero_tail": D.Synth(1258, seed=12, scan="end", pad=0),
    "overlap": D.Synth(1252, seed=13, scan="overlap"),
    "shuffle": D.Synth(1258, seed=14, scan="shuffle"),
    "short_mb_height": D.Synth(1252, seed=15, mb_height=7),
    "sar": D.Synth(1259, seed=16, header_width=1280, mb_height=9),
    "fields_same_cur_field": D.Synth(1243, seed=17, fields=(1, 1), mb_height=5),
    "fields_bff": D.Synth(1241, seed=18, fields=(1, 0), mb_height=5),
    "row_reads_second_field": D.Synth(1243, seed=19, scan="cu_end", mb_height=4),
}

_synth_cache = {}


def synth(dref, name):
    if name not in _synth_cache:
        _synth_cache[name] = D.synth(dref, SYNTH[name])
    return _synth_cache[name]


@pytest.mark.parametrize("name", sorted(REAL))
def test_real_packets(hs, dref, eref, name):
    cid, contents, il, mbd = REAL[name]
    D.check(hs, dref, PU.HostMem(), D.real_packets(eref, cid, contents, interlaced=il, mb_decision=mbd, seed=7 + len(name)))


@pytest.mark.parametrize("name", sorted(SYNTH))
def test_synthesised_packets(hs, dref, name):
    D.check(hs, dref, PU.HostMem(), [synth(dref, name)])


def test_reachability(hs, dref):
    """the damaged-block break, the int16 truncation of dequantised levels and the zero-bit tail are reached by the cases above.  The
    32-bit wrap of (2 level + 1) qscale weight needs a weight of at least 129 at 10 bit; the weights of ff_dnxhd_cid_table stop at 94
    there, so with the reference's own table the product peaks at 0.73 * 2^31; test_dequantisation_wraps_with_caller_weights reaches the
    wrap with a caller's table."""
    assert D.check(hs, dref, PU.HostMem(), [synth(dref, "damaged_runs")]) > 0
    _, _, ent = D.cid_table(dref)
    e = ent[1250]
    w = max(D.u8(e.luma_weight, 64).max(), D.u8(e.chroma_weight, 64).max())
    T = D.codes(e)
    top = max(int(T["ac_level"][k]) + (63 << 6 if T["ac_index"][k] else 0) for k in range(257) if T["ac_bits"][k])
    assert ((2 * top + 1) * 2047 * int(w) + 8) >> 4 > 32767                   # wrap_10bit's largest levels are truncated to int16
    assert (2 * top + 1) * 2047 * 129 >= 1 << 31 > (2 * top + 1) * 2047 * 128     # a weight of 129 would wrap
    pkt = synth(dref, "zero_tail")
    assert int.from_bytes(pkt[0x170 + 4 * 44:0x174 + 4 * 44], "big") + 0x280 == len(pkt)           # the last of 45 rows


def test_gray_and_padded_linesizes(hs, dref, eref):
    pk = D.real_packets(eref, 1251, ["natural"], seed=3)
    D.check(hs, dref, PU.HostMem(), pk, gray=1)
    D.check(hs, dref, PU.HostMem(), pk + [synth(dref, "444")], pad=40)


def test_mixed_cids_one_call(hs, dref, eref):
    pk = D.real_packets(eref, 1235, ["natural"], seed=4) + [synth(dref, n) for n in ("444", "mbaff_1260", "sar", "fields_bff")] + \
        D.real_packets(eref, 1243, ["noise"], seed=5)
    D.check(hs, dref, PU.HostMem(), pk)


def malformed(dref, eref):
    """(name, packet) pairs that dnxhd_decode_header or ff_set_dimensions refuse"""
    base = bytearray(D.real_packets(eref, 1252, ["flat"], seed=9)[0])
    il = bytearray(D.real_packets(eref, 1243, ["flat"], seed=9)[0])
    out = [("short", bytes(base[:0x27f])), ("unit_short", bytes(base[:0x300]))]
    for name, off, val in (("prefix", 4, 3), ("depth", 0x21, 0x40), ("cid", 0x2b, 0x99), ("mbh", 0x16d, 69), ("mbh_tall", 0x16d, 60),
                           ("scan", 0x170, 0x7f)):
        b = bytearray(base); b[off] = val; out.append((name, bytes(b)))
    b = bytearray(base); b[0x18:0x1a] = b"\0\0"; b[0x16d] = 0; out.append(("height0", bytes(b)))
    out.append(("second_unit_short", bytes(il[:len(il) // 2 + 0x100])))
    b = bytearray(il); b[len(il) // 2 + 0x21] = 0x10; out.append(("second_unit_depth", bytes(b)))
    return out


def test_probe_matches_reference_return_codes(hs, dref, eref):
    cids, n, _ = D.cid_table(dref)
    for name, pkt in malformed(dref, eref):
        ret, info = D.info_of(hs, pkt, cids, n)
        planes = [np.zeros((2200, 4096), np.uint8) for _ in range(3)]
        arr = (C.c_void_p * 3)(*[p.ctypes.data for p in planes])
        ls = (C.c_int * 3)(4096, 4096, 4096)
        buf = np.frombuffer(pkt, np.uint8).copy()
        want = dref.ref_dnxhd_decode(buf.ctypes.data, len(pkt), 0, arr, ls, 2200, None, None)
        assert ret == want and ret < 0, (name, ret, want)


def refusal_packets(dref, eref):
    """(name, packet, cid table mutation) the probe refuses with -1"""
    base = D.real_packets(eref, 1252, ["flat"], seed=9)[0]
    il = D.real_packets(eref, 1243, ["flat"], seed=9)[0]
    out = []
    b = bytearray(base); b[0x28:0x2c] = b"\0\0\0\0"; out.append(("cid0", bytes(b)))
    b = bytearray(base); b[0x21] = 0x58; out.append(("depth_vs_entry", bytes(b)))
    b = bytearray(base); b[0x170:0x174] = (0xffffff00).to_bytes(4, "big"); out.append(("scan_wrap", bytes(b)))
    h = len(il) // 2
    b = bytearray(il); b[h + 5] = 1; out.append(("second_not_interlaced", bytes(b)))
    b = bytearray(il); b[h + 0x28:h + 0x2c] = (1253).to_bytes(4, "big"); out.append(("second_cid", bytes(b)))
    b = bytearray(il); b[h + 0x18:h + 0x1a] = (100).to_bytes(2, "big"); b[h + 0x16d] = 2; out.append(("second_size", bytes(b)))
    return out


def many_subtable_code():
    """(codes, lengths) of 257 AC symbols: a complete canonical prefix code whose 10-bit codes sit under 25 different 9-bit prefixes (codes
    of lengths 1, 2, 3, 4, 7, 8, 9 and fifty of 10; the other symbols have none)"""
    lens = [1, 2, 3, 4, 7, 8, 9] + [10] * 50
    codes, code, prev = [], 0, lens[0]
    for k, n in enumerate(lens):
        if k:
            code = (code + 1) << (n - prev)
        codes.append(code)
        prev = n
    assert sum(2.0 ** -n for n in lens) == 1.0 and len({c >> 1 for c, n in zip(codes, lens) if n == 10}) == 25
    return codes + [0] * (257 - len(codes)), lens + [0] * (257 - len(lens))


def test_dequantisation_wraps_with_caller_weights(hs, dref):
    """The 32-bit wrap of (2 level + 1) qscale weight, which the weights of ff_dnxhd_cid_table cannot reach: CID 1250's entry with every
    weight 255, qscale 2047 and the largest levels.  The reference decoder cannot take another table, so the product's dequantised blocks
    (the entropy stage's workspace, per row, macroblock and block) are compared with the synthesiser's model of dnxhd_decode_dct_block."""
    _, _, ent = D.cid_table(dref)
    w255 = (C.c_uint8 * 64)(*([255] * 64))
    for is444, cid in ((False, 1250), (True, 1256)):
        s = D.Synth(cid, seed=70, qscales=(2047, 1500), big=0.6, eob=0.15, runs=0.0, mb_height=2, is444=is444,
                    weights=(np.full(64, 255), np.full(64, 255)))
        e = tables.FFDnxhdCidEntry.from_buffer_copy(ent[cid])
        e.luma_weight = e.chroma_weight = C.cast(w255, C.c_void_p)
        tab = (tables.FFDnxhdCidEntry * 1)(e)
        pkt = np.frombuffer(D.synth(dref, s), np.uint8).copy()
        assert s.wraps > 100
        mem = PU.HostMem()
        info = tables.FFDnxhdFrameInfo()
        assert hs.ff_dnxhd_probe_cuda(pkt.ctypes.data, len(pkt), C.cast(tab, C.c_void_p), 1, C.byref(info)) == 0
        w = tables.FFDnxhdDecodeWork()
        w.pkt_host, w.pkt, w.size = pkt.ctypes.data, mem.put(pkt), len(pkt)
        for p in range(3):
            w.data[p], w.linesize[p], w.lines[p] = mem.put(np.zeros(info.lines * 4096, np.uint8)), 4096, info.lines
        arr = (tables.FFDnxhdDecodeWork * 1)(w)
        need = hs.ff_dnxhd_decode_workspace_cuda(arr, 1, C.cast(tab, C.c_void_p), 1)
        ws = mem.put(np.zeros(need, np.uint8))
        assert hs.ff_dnxhd_decode_frames_cuda(arr, 1, C.cast(tab, C.c_void_p), 1, C.c_void_p(ws), need, None) == 0
        got = mem.get(ws, np.int16, s.expected.shape)
        assert np.array_equal(got, s.expected), np.argwhere(got != s.expected)[:4]


def test_refusals(hs, dref, eref):
    check_refusals(hs, dref, eref, PU.HostMem())


def check_refusals(lib, dref, eref, mem):
    cids, n, ent = D.cid_table(dref)
    for name, pkt in refusal_packets(dref, eref):
        ret, _ = D.info_of(lib, pkt, cids, n)
        assert ret == -1 and lib.avb200_last_error(), name
        lib.avb200_clear_error()
    # CID entries with a broken code: a copy of 1258's entry with one AC / run / DC length changed, or a DC code past 7 bits
    pkt = D.real_packets(eref, 1258, ["flat"], seed=9)[0]
    e = ent[1258]
    many = many_subtable_code()
    for field, count, idx, val in (("ac_bits", 257, 3, 0), ("run_bits", 62, 5, 1), ("dc_bits", 12, 0, 8), ("ac_bits", 257, 0, 17),
                                   ("ac_codes", 257, None, None)):
        mut = tables.FFDnxhdCidEntry.from_buffer_copy(e)
        if idx is None:                                       # a complete code that needs 25 second-level tables
            codes16, bits8 = (C.c_uint16 * 257)(*many[0]), (C.c_uint8 * 257)(*many[1])
            mut.ac_codes, mut.ac_bits = C.cast(codes16, C.c_void_p), C.cast(bits8, C.c_void_p)
        else:
            arr = (C.c_uint8 * count)(*D.u8(getattr(e, field), count))
            arr[idx] = val
            setattr(mut, field, C.cast(arr, C.c_void_p))
        one = (tables.FFDnxhdCidEntry * 1)(mut)
        info = tables.FFDnxhdFrameInfo()
        assert lib.ff_dnxhd_probe_cuda(pkt, len(pkt), C.cast(one, C.c_void_p), 1, C.byref(info)) == -1 and lib.avb200_last_error(), field
        lib.avb200_clear_error()
        works_pkt = np.frombuffer(pkt, np.uint8).copy()
        w = tables.FFDnxhdDecodeWork()
        w.pkt_host, w.pkt, w.size = works_pkt.ctypes.data, mem.put(works_pkt), len(pkt)
        planes = [mem.put(np.zeros(1100 * 2048, np.uint8)) for _ in range(3)]
        for p in range(3):
            w.data[p], w.linesize[p], w.lines[p] = planes[p], 2048, 1100
        arrw = (tables.FFDnxhdDecodeWork * 1)(w)
        assert lib.ff_dnxhd_decode_workspace_cuda(arrw, 1, C.cast(one, C.c_void_p), 1) == 0, field
        lib.avb200_clear_error()
        ws = mem.put(np.zeros(64 << 20, np.uint8))
        rc = lib.ff_dnxhd_decode_frames_cuda(arrw, 1, C.cast(one, C.c_void_p), 1, C.c_void_p(ws), 64 << 20, None)
        assert rc == -1 and lib.avb200_last_error(), field
        lib.avb200_clear_error()
    # planes and workspace
    base = D.real_packets(eref, 1252, ["flat"], seed=9)[0]
    muts = [lambda w: setattr(w, "pkt", None), lambda w: w.data.__setitem__(0, None), lambda w: w.linesize.__setitem__(0, 0),
            lambda w: w.linesize.__setitem__(1, 10), lambda w: w.lines.__setitem__(2, 700), lambda w: w.linesize.__setitem__(2, w.linesize[1] + 2)]
    for k, m in enumerate(muts):
        rc, _, _ = D.run(lib, mem, [base], cids, n, mutate=m)
        assert rc == -1 and lib.avb200_last_error(), k
        lib.avb200_clear_error()
    rc, _, _ = D.run(lib, mem, [base], cids, n, ws_delta=-1)
    assert rc == -1
    lib.avb200_clear_error()


def test_workspace_query(hs, dref, eref):
    cids, n, _ = D.cid_table(dref)
    pkt = np.frombuffer(D.real_packets(eref, 1252, ["flat"], seed=9)[0], np.uint8).copy()
    w = tables.FFDnxhdDecodeWork()
    w.pkt_host, w.pkt, w.size = pkt.ctypes.data, pkt.ctypes.data, len(pkt)
    for p in range(3):
        w.data[p], w.linesize[p], w.lines[p] = pkt.ctypes.data, 1280, 720
    arr = (tables.FFDnxhdDecodeWork * 2)(w, w)
    one = hs.ff_dnxhd_decode_workspace_cuda(arr, 1, cids, n)
    assert one >= 45 * 80 * 8 * 128 and hs.ff_dnxhd_decode_workspace_cuda(arr, 2, cids, n) == 2 * one
    assert hs.ff_dnxhd_decode_workspace_cuda(arr, 0, cids, n) == 0


def test_header_exports_and_ctypes_agree(hs, dref):
    import os
    import re
    hdr = open(os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "include", "avdsp_b200.h")).read()
    fm = np.zeros(3, np.int32)
    dref.ref_dnxhd_pix_fmts(fm.ctypes.data)
    got = [int(re.search(r"#define FF_DNXHD_PIX_FMT_%s\s+(\d+)" % n, hdr).group(1)) for n in ("YUV422P", "YUV422P10", "YUV444P10")]
    assert got == list(fm)
    for s, fields in (("FFDnxhdFrameInfo", tables.FFDnxhdFrameInfo._fields_), ("FFDnxhdDecodeWork", tables.FFDnxhdDecodeWork._fields_)):
        body = re.search(r"typedef struct %s \{(.*?)\} %s;" % (s, s), hdr, re.S).group(1)
        body = re.sub(r"/\*.*?\*/", "", body, flags=re.S)
        names = re.findall(r"(\w+)(?:\[\d\])?\s*[,;]", body)
        assert names == [f[0] for f in fields], (s, names)
    for name in ("ff_dnxhd_probe_cuda", "ff_dnxhd_decode_workspace_cuda", "ff_dnxhd_decode_frames_cuda"):
        assert name in hdr and hasattr(hs, name)
