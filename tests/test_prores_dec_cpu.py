"""The ProRes decoder (libav_b200/csrc/prores_dec.cu + prores_dec.cuh, with prores.cu's picture kernel) compiled as host C++
(tests/hostsim/prores_dec_hostsim.cpp) against the reference decoder with the checked reader (oracle/_ref/libproresdecref.so:
proresdec.c, unmodified), one fresh context per packet: every plane byte for byte, the alpha plane and the sentinel in what the decoder
does not write included, and the probe's return value and frame info.  Packets from the reference encoder (every profile and format,
both field orders, every slice width, odd sizes) and header edits of them (matrices, scale factors, slice header sizes, short, zero,
zero-filled, truncated and bit-flipped planes, yuva422p10, bad frame and picture headers), the probe's return codes, and every refusal.

The host build's >> masks its count as x86 does, so the undefined shift of decode_vlc_codeword (zero_plane_dc_* cases) is told apart
from CUDA's >> only on the GPU (tests/test_gpu_prores_dec.py runs the same cases).

Mutations of prores_dec.cuh / prores_dec.cu / prores.cuh this file catches (failed tests of 72): no clamp of the reader's position 16;
zeros instead of the packet's bytes past a plane's end 18; the shift without its mask, written with CUDA's result for counts past 31
(`len > 32 ? 0 : buf >> (32 - len)`) 4; writing the planes after a failed one 7; writing alpha after a failed chroma plane 5; no
MAX_PADDING test 62; right-edge slices not limited to the slice width (prd_slice_pos without `b >= swf`): the first 7-macroblock case
writes past its blocks and the host process aborts."""
import ctypes as C
import random

import numpy as np
import pytest

import hostsim_build
import prores_util as PU
import prores_enc_util as E
import prores_dec_util as D
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


F422, F444, F4444 = E.FMT_422, E.FMT_444, E.FMT_4444

# name -> encode() arguments: every profile, the three formats with 8- and 16-bit alpha, both field orders, every slice width at 112
# samples (7 macroblocks: right-edge slices of 4, 2 and 1 macroblocks at 8 and 4 per slice, of 1 at 2 per slice), progressive and
# interlaced, odd progressive and interlaced heights
REAL = {
    "proxy": (F422, 64, 48, 0, 0), "lt": (F422, 64, 48, 0, 1), "standard": (F422, 64, 48, 0, 2), "hq": (F422, 64, 48, 0, 3),
    "4444_a16": (F4444, 64, 48, 0, 4), "4444_a8": (F4444, 48, 32, 0, 4, 8, dict(alpha_bits=8)),
    "444": (F444, 64, 32, 0, 3), "tff": (F422, 80, 64, 1, 2), "bff": (F422, 80, 64, 2, 3), "4444_bff": (F4444, 48, 64, 2, 4),
    "mps1": (F422, 112, 32, 0, 2, 1), "mps2": (F444, 112, 32, 0, 2, 2), "mps4": (F422, 112, 32, 0, 2, 4), "mps8_edges": (F4444, 112, 32, 0, 4, 8),
    "mps2_il": (F4444, 112, 64, 1, 4, 2), "mps4_il": (F444, 112, 64, 2, 3, 4), "mps8_il": (F422, 112, 64, 1, 2, 8),
    "odd_height": (F422, 72, 37, 0, 2), "odd_height_il": (F444, 72, 37, 1, 2), "noise": (F422, 64, 48, 0, 0, 8, dict(content="noise")),
}

_cache = {}


def real(eref, name):
    if name not in _cache:
        a = REAL[name]
        fmt, w, h, il, prof = a[:5]
        mps = a[5] if len(a) > 5 else 8
        kw = a[6] if len(a) > 6 else {}
        _cache[name] = D.encode(eref, fmt, w, h, interlaced=il, profile=prof, mbs_per_slice=mps, seed=len(name), **kw)
    return _cache[name]


def _flips(b, P, seed, n):
    r = random.Random(seed)
    sl = [s for pic in P["pics"] for s in pic["slices"]]
    for _ in range(n):
        off, size = r.choice(sl)
        k = off + r.randrange(max(size, 1))
        b[k] ^= 1 << r.randrange(8)


def _short_slice(b, P):
    """the first slice is 3 bytes and the second takes the rest of both"""
    pic = P["pics"][0]
    a, c = D.rb16(b, pic["index"]), D.rb16(b, pic["index"] + 2)
    D.set16(b, pic["index"], 3)
    D.set16(b, pic["index"] + 2, a + c - 3)


def _plane_sizes(b, P, fn):
    for pic in P["pics"]:
        for k, (off, size) in enumerate(pic["slices"]):
            fn(b, off, size, k)


def _small_frame_header(b, P):
    """frame hdr_size 16: the picture header starts at the frame header's byte 16, so bytes 16..19 (colour space, alpha_info, flags) are
    the picture header's first four bytes; decode_frame_header still reads its bytes 8..19"""
    pic = P["pics"][0]
    ph = bytearray(b[pic["at"]:])
    ps = D.rb32(ph, 1) & ~0x0300                                     # a smaller pic_data_size whose third byte has flags 0
    D.set32(ph, 1, ps)
    out = bytearray(b[:24]) + ph
    D.set16(out, 8, 16)
    out[24:28] = ph[0:4]
    D.set32(out, 0, len(out))
    return out


def _second_header(b, P, v):
    b[P["pics"][1]["at"]] = v


EDITS = {
    # frame header
    "matrices_flags0": ("hq", lambda b, P: b.__setitem__(27, 0)),
    "matrices_flags1": ("hq", lambda b, P: b.__setitem__(27, 1)),
    "matrices_flags2": ("hq", lambda b, P: b.__setitem__(27, 2)),
    "matrices_custom3": ("standard", lambda b, P: b.__setitem__(slice(28, 156), bytes(random.Random(3).randrange(0, 256) for _ in range(128)))),
    "small_frame_header": ("standard", _small_frame_header),
    "yuva422": ("4444_a16", lambda b, P: b.__setitem__(20, (b[20] & 0x3f) | 0x80)),
    "yuva422_a8": ("4444_a8", lambda b, P: b.__setitem__(20, (b[20] & 0x3f) | 0x80)),
    "alpha_on_422": ("hq", lambda b, P: b.__setitem__(25, (b[25] & 0xf0) | 2)),
    # picture headers
    "pic_data_size0": ("tff", lambda b, P: D.set32(b, P["pics"][0]["at"] + 1, 0)),
    "pic_data_size_neg_second": ("bff", lambda b, P: D.set32(b, P["pics"][1]["at"] + 1, 0x80000000)),
    "pic_data_size_neg_first": ("tff", lambda b, P: D.set32(b, P["pics"][0]["at"] + 1, 0xfffffff0)),
    "second_header_small": ("tff", lambda b, P: _second_header(b, P, 0x20)),
    "second_slice_count": ("bff", lambda b, P: D.set16(b, P["pics"][1]["at"] + 5, P["pics"][1]["n"] + 1)),
    "second_out_of_data": ("tff", lambda b, P: D.set16(b, P["pics"][1]["index"], 0xffff)),
    "second_swf": ("4444_bff", lambda b, P: b.__setitem__(P["pics"][1]["at"] + 7, 0x40)),
    # slices
    "sf_bytes": ("standard", lambda b, P: _plane_sizes(b, P, lambda b, o, s, k: b.__setitem__(o + 1, (0, 1, 128, 129, 224, 255)[k % 6]))),
    "slice_hdr_5": ("standard", lambda b, P: _plane_sizes(b, P, lambda b, o, s, k: b.__setitem__(o, 5 << 3) if k % 2 else None)),
    "slice_hdr_7": ("hq", lambda b, P: _plane_sizes(b, P, lambda b, o, s, k: b.__setitem__(o, 7 << 3) if k % 2 else None)),
    "slice_hdr_8": ("hq", lambda b, P: _plane_sizes(b, P, lambda b, o, s, k: b.__setitem__(o, 8 << 3) if k % 3 == 1 else None)),
    "slice_hdr_31": ("4444_a16", lambda b, P: _plane_sizes(b, P, lambda b, o, s, k: b.__setitem__(o, 31 << 3) if k % 3 == 2 else None)),
    "short_slice": ("hq", _short_slice),
    "zero_size_y": ("hq", lambda b, P: _plane_sizes(b, P, lambda b, o, s, k: D.set16(b, o + 2, 0) if k % 2 == 0 else None)),
    "zero_size_u": ("4444_a16", lambda b, P: _plane_sizes(b, P, lambda b, o, s, k: D.set16(b, o + 4, 0) if k % 2 else None)),
    "truncated_y": ("hq", lambda b, P: _plane_sizes(b, P, lambda b, o, s, k: D.set16(b, o + 2, D.rb16(b, o + 2) // (k % 4 + 2)))),
    "y_too_large": ("standard", lambda b, P: _plane_sizes(b, P, lambda b, o, s, k: D.set16(b, o + 2, s) if k % 2 else None)),
    "alpha_sizes": ("4444_a8", lambda b, P: _plane_sizes(b, P, lambda b, o, s, k: (b.__setitem__(o, 8 << 3), D.set16(b, o + 6, k % 5)))),
    "bit_flips": ("proxy", lambda b, P: _flips(b, P, 1, 60)),
    "bit_flips_444": ("444", lambda b, P: _flips(b, P, 2, 80)),
    "bit_flips_alpha": ("4444_a16", lambda b, P: _flips(b, P, 3, 200)),
    "bit_flips_il": ("tff", lambda b, P: _flips(b, P, 4, 80)),
}
for _lead in (0, 10, 14, 20, 26, 27, 28, 29, 30, 31, 33, 40):
    # one plane of every slice zero-filled after one 1 bit: DC decoding (no end guard) reaches exp-Golomb lengths past 32.  In a plane of 4
    # to 6 bytes the first DC code's value shows (27..30 leading zeros: the count modulo 32 keeps 1 to 3 bits where CUDA's >> gives 0); in
    # a whole plane the AC codes that follow fail
    EDITS["zero_plane_dc_%d" % _lead] = ("hq", lambda b, P, L=_lead: _plane_sizes(
        b, P, lambda b, o, s, k: D.zero_dc_run(b, (o, s), k % 3, L + k % 2, None if k % 3 == 2 else 4 + k % 3)))
EDITS["zero_planes_all"] = ("4444_a16", lambda b, P: _plane_sizes(b, P, lambda b, o, s, k: [D.zero_dc_run(b, (o, s), p, 99) for p in range(3)]))

_ecache = {}


def edited(eref, name):
    if name not in _ecache:
        base, fn = EDITS[name]
        _ecache[name] = D.edit(real(eref, base), name, fn)
    return _ecache[name]


def malformed(eref):
    """(name, packet) pairs that decode_frame refuses before get_buffer"""
    base = real(eref, "hq")
    out = [("short", D.Pkt(base.data[:27], base.w, base.h)),
           ("atom_size", D.edit(base, "atom", lambda b, P: D.set32(b, 0, len(b) + 1))),
           ("frame_id", D.edit(base, "id", lambda b, P: b.__setitem__(4, ord("x")))),
           ("width", D.Pkt(base.data, base.w + 1, base.h)), ("height", D.Pkt(base.data, base.w, base.h - 1)),
           ("hdr_size", D.edit(base, "hdr", lambda b, P: D.set16(b, 8, len(b)))),
           ("version2", D.edit(base, "v2", lambda b, P: D.set16(b, 10, 2))),
           ("frame_type3", D.edit(base, "ft3", lambda b, P: b.__setitem__(20, b[20] | 12))),
           ("alpha_info3", D.edit(base, "a3", lambda b, P: b.__setitem__(25, (b[25] & 0xf0) | 3))),
           ("chroma0", D.edit(base, "cf0", lambda b, P: b.__setitem__(20, b[20] & 0x3f))),
           ("chroma1", D.edit(base, "cf1", lambda b, P: b.__setitem__(20, (b[20] & 0x3f) | 0x40))),
           ("luma_matrix_short", D.edit(base, "lm", lambda b, P: (b.__setitem__(27, 3), D.set16(b, 8, 83)))),
           ("chroma_matrix_short", D.edit(base, "cm", lambda b, P: (b.__setitem__(27, 3), D.set16(b, 8, 147))))]
    return out


def first_header_failures(eref):
    """(name, packet) pairs whose first picture header fails after get_buffer: nothing is written, decode_frame returns INVALIDDATA"""
    base = real(eref, "hq")
    at = D.parse(base)["pics"][0]["at"]
    return [("pic_hdr_small", D.edit(base, "ph", lambda b, P: b.__setitem__(at, 7 << 3))),
            ("pic_data_size", D.edit(base, "pds", lambda b, P: D.set32(b, at + 1, len(b)))),
            ("swf4", D.edit(base, "swf", lambda b, P: b.__setitem__(at + 7, 0x40))),
            ("shf", D.edit(base, "shf", lambda b, P: b.__setitem__(at + 7, 0x31))),
            ("slice_count", D.edit(base, "n", lambda b, P: D.set16(b, at + 5, P["pics"][0]["n"] - 1))),
            ("slice_table_short", D.edit(base, "tbl", lambda b, P: _truncate(b, P["pics"][0]["index"] + 3))),
            ("out_of_slice_data", D.edit(base, "oos", lambda b, P: D.set16(b, P["pics"][0]["index"], D.rb16(b, P["pics"][0]["index"]) + 1)))]


def _truncate(b, n):
    out = bytearray(b[:n])
    D.set32(out, 0, n)
    return out


@pytest.mark.parametrize("name", sorted(REAL))
def test_reference_encoder_packets(hs, dref, eref, name):
    D.check(hs, dref, PU.HostMem(), [real(eref, name)])


@pytest.mark.parametrize("name", sorted(EDITS))
def test_header_edits(hs, dref, eref, name):
    D.check(hs, dref, PU.HostMem(), [edited(eref, name)])


def test_edits_reach_their_cases(hs, dref, eref):
    """the edits above reach what they are named for: a failing plane, a second picture that fails, a first pic_data_size of 0"""
    assert D.probe(hs, edited(eref, "second_header_small"))[1].pictures == 1
    assert D.probe(hs, edited(eref, "second_header_small"))[1].result == D.INVALIDDATA
    assert D.probe(hs, edited(eref, "pic_data_size_neg_first"))[1].pictures == 0
    assert D.probe(hs, edited(eref, "pic_data_size0"))[1].pictures == 2
    assert D.probe(hs, edited(eref, "yuva422"))[1].pix_fmt == tables_fmt(2)
    assert D.parse(edited(eref, "small_frame_header"))["hdr"] == 16


def tables_fmt(k):
    return D.tables_pix_fmts()[k]


def test_batch_of_every_case(hs, dref, eref):
    """one call over packets of every format, field order and size"""
    pk = [real(eref, n) for n in ("hq", "4444_a8", "bff", "mps1", "odd_height_il")] + [edited(eref, n) for n in ("bit_flips_alpha", "yuva422")]
    for p in pk:
        D.check(hs, dref, PU.HostMem(), [p])
    by_size = {}
    for p in pk:
        by_size.setdefault((p.w, p.h), []).append(p)
    for group in by_size.values():
        D.check(hs, dref, PU.HostMem(), group, pad=40)


def test_fresh_context_equals_one_context(hs, dref, eref):
    """a mixed sequence through ONE reference context gives the planes fresh contexts give: qmat_* are rewritten per frame and
    prev_slice_sf is reset per picture, so the call needs no context"""
    seq = [real(eref, "hq"), edited(eref, "matrices_custom3"), real(eref, "proxy"), edited(eref, "matrices_flags0"), edited(eref, "sf_bytes"),
           real(eref, "hq")]
    lines = [D.probe(hs, p)[1].lines + 16 for p in seq]
    one, rows = D.ref_decode(dref, seq, lines)
    for k, p in enumerate(seq):
        fresh, frow = D.ref_decode(dref, [p], [lines[k]])
        assert list(rows[k]) == list(frow[0]), k
        for a, b in zip(one[k], fresh[0]):
            assert np.array_equal(a, b), k


def test_probe_matches_reference(hs, dref, eref):
    for name, pkt in malformed(eref):
        ret, _ = D.probe(hs, pkt)
        assert ret == D.INVALIDDATA, (name, ret)
        assert D.check_probe(hs, dref, pkt) is None, name
    for name, pkt in first_header_failures(eref):
        info = D.check_probe(hs, dref, pkt)
        assert info is not None and info.pictures == 0 and info.result == D.INVALIDDATA, name
        D.check(hs, dref, PU.HostMem(), [pkt])


def test_undefined_shift_is_reached_and_masked(hs, dref):
    """the reference as compiled shifts by 32 - len modulo 32 (x86-64's shr) for len > 32; the zero_plane_dc_* cases reach such lengths"""
    for a, s in ((0x12345678, 36), (0xdeadbeef, 60), (31, 68), (0x80000000, 33)):
        assert dref.ref_prores_dec_neg_usr32(a, s) == (a >> ((32 - s) & 31)), (a, s)


def test_tables_agree(hs, dref):
    a, b = np.zeros(256, np.int32), np.zeros(256, np.int32)
    na, nb = dref.ref_prores_dec_tables(a.ctypes.data), hs.hostsim_prores_dec_tables(b.ctypes.data)
    assert na == nb == 166 and np.array_equal(a[:na], b[:nb])


def test_pix_fmts_and_ctypes_agree(hs, dref):
    import os
    import re
    hdr = open(os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "include", "avdsp_b200.h")).read()
    fm = np.zeros(4, np.int32)
    dref.ref_prores_dec_pix_fmts(fm.ctypes.data)
    got = [int(re.search(r"#define FF_PRORES_PIX_FMT_%s\s+(\d+)" % n, hdr).group(1)) for n in ("YUV422P10", "YUV444P10", "YUVA422P10", "YUVA444P10")]
    assert got == list(fm) == list(D.tables_pix_fmts())
    for s, fields in (("FFProresFrameInfo", tables.FFProresFrameInfo._fields_), ("FFProresDecodeWork", tables.FFProresDecodeWork._fields_)):
        body = re.search(r"typedef struct %s \{(.*?)\} %s;" % (s, s), hdr, re.S).group(1)
        body = re.sub(r"/\*.*?\*/", "", body, flags=re.S)
        names = re.findall(r"(\w+)(?:\[\d\])?\s*[,;]", body)
        assert names == [f[0] for f in fields], (s, names)


def check_refusals(lib, dref, eref, mem):
    base, alpha = real(eref, "hq"), real(eref, "4444_a16")
    # a packet the probe refuses, and a zero height
    for pkt in (D.edit(base, "id", lambda b, P: b.__setitem__(4, 0)),):
        hb = np.frombuffer(pkt.data, np.uint8).copy()
        w = tables.FFProresDecodeWork(pkt_host=hb.ctypes.data, pkt=mem.put(hb), size=len(hb), width=pkt.w, height=pkt.h)
        for p in range(4):
            w.data[p], w.linesize[p], w.lines[p] = mem.put(np.zeros(64 * 1024, np.uint8)), 1024, 64
        arr = (tables.FFProresDecodeWork * 1)(w)
        assert lib.ff_prores_decode_workspace_cuda(arr, 1) == 0
        assert lib.ff_prores_decode_frames_cuda(arr, 1, C.c_void_p(mem.put(np.zeros(1 << 20, np.uint8))), 1 << 20, None) == -1
        lib.avb200_clear_error()
    zero = D.Pkt(D.edit(base, "h0", lambda b, P: D.set16(b, 18, 0)).data, base.w, 0)
    assert D.probe(lib, zero)[0] == -1 and lib.avb200_last_error()
    lib.avb200_clear_error()
    muts = [lambda w: setattr(w, "pkt", None), lambda w: w.data.__setitem__(0, None), lambda w: w.data.__setitem__(1, w.data[1] + 1),
            lambda w: w.linesize.__setitem__(0, 0), lambda w: w.linesize.__setitem__(1, w.linesize[1] - 1),
            lambda w: w.linesize.__setitem__(0, 16 * ((base.w + 15) // 16) * 2 - 2), lambda w: w.lines.__setitem__(2, w.lines[2] - 1),
            lambda w: w.linesize.__setitem__(2, -64)]
    for k, m in enumerate(muts):
        rc, _, _ = D.run(lib, mem, [base], mutate=m)
        assert rc == -1 and lib.avb200_last_error(), k
        lib.avb200_clear_error()
    for k, m in enumerate([lambda w: w.data.__setitem__(3, None), lambda w: w.lines.__setitem__(3, 1)]):
        rc, _, _ = D.run(lib, mem, [alpha], mutate=m)
        assert rc == -1 and lib.avb200_last_error(), ("alpha", k)
        lib.avb200_clear_error()
    rc, _, _ = D.run(lib, mem, [base], mutate=lambda w: w.data.__setitem__(3, None))        # no alpha plane is needed without alpha
    assert rc == 0
    rc, _, _ = D.run(lib, mem, [base], ws_delta=-1)
    assert rc == -1 and lib.avb200_last_error()
    lib.avb200_clear_error()
    rc, _, _ = D.run(lib, mem, [base], ws_offset=8)                  # a workspace that is not 16-byte aligned
    assert rc == -1 and lib.avb200_last_error()
    lib.avb200_clear_error()
    assert lib.ff_prores_decode_frames_cuda(None, 1, None, 0, None) == -1
    lib.avb200_clear_error()
    assert lib.ff_prores_decode_frames_cuda(None, 0, None, 0, None) == 0


def test_refusals(hs, dref, eref):
    check_refusals(hs, dref, eref, PU.HostMem())


def test_workspace_query(hs, dref, eref):
    pkt = real(eref, "tff")
    hb = np.frombuffer(pkt.data, np.uint8).copy()
    w = tables.FFProresDecodeWork(pkt_host=hb.ctypes.data, pkt=hb.ctypes.data, size=len(hb), width=pkt.w, height=pkt.h)
    for p in range(4):
        w.data[p], w.linesize[p], w.lines[p] = hb.ctypes.data & ~1, 1024, 64
    arr = (tables.FFProresDecodeWork * 2)(w, w)
    one = hs.ff_prores_decode_workspace_cuda(arr, 1)
    assert one >= 2 * 5 * 2 * 8 * 128 and hs.ff_prores_decode_workspace_cuda(arr, 2) == 2 * one        # two fields of 5 x 2 macroblocks
    assert hs.ff_prores_decode_workspace_cuda(arr, 0) == 0 and hs.ff_prores_decode_workspace_cuda(None, 1) == 0
