"""The ProRes encoder (libav_b200/csrc/prores_enc.cu + prores_enc.cuh) compiled as host C++ (tests/hostsim/prores_enc_hostsim.cpp) against
the reference encoder (oracle/_ref/libproresencref.so: proresenc.c, unmodified): whole packets byte for byte and every slice's quantiser
over formats, profiles, field orders, slice widths, edge geometries, every option and content that takes every path of the rate control.
Also the restated tables against the reference's, every refusal, the workspace query, and the public header against the library's exports
and the ctypes mirrors."""
import ctypes as C
import os
import re
import subprocess

import numpy as np
import pytest

import hostsim_build
import prores_util as PU
import prores_enc_util as E
from libav_b200 import tables

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)


@pytest.fixture(scope="session")
def eref(built):
    lib = E.ref()
    if lib is None:
        pytest.skip("oracle/_ref not built (no reference tree in this environment)")
    return lib


@pytest.fixture(scope="session")
def hs(built):
    return hostsim_build.load()


def encode_and_compare(hs, eref, cases):
    rc, pkts, sizes, _ = E.run(hs, PU.HostMem(), cases)
    assert rc == 0, hs.avb200_last_error()
    out = []
    for c, got in zip(cases, pkts):
        want, wq = E.ref_encode(eref, c)
        E.compare(c, got, want, wq)
        out.append(got)
    return out


GROUPS = {"matrix": E.matrix_cases, "edges": E.edge_cases, "options": E.option_cases, "content": E.content_cases}


@pytest.mark.parametrize("group", sorted(GROUPS))
def test_packets_match_reference_encoder(hs, eref, group):
    """every case of the group in one call; each packet equals encode_frame's, each slice's quantiser find_quant_thread's"""
    encode_and_compare(hs, eref, GROUPS[group]())


def test_matrix_covers_every_pair():
    """formats x profiles x field orders x mbs_per_slice: every pair of values occurs together"""
    rows = {(c.fmt, c.profile, c.interlaced, c.mbs_per_slice) for c in E.matrix_cases()}
    values = [[0, 1, 2], [0, 1, 2, 3, 4], [0, 1, 2], [1, 2, 4, 8]]
    for i in range(4):
        for j in range(i + 1, 4):
            for a in values[i]:
                for b in values[j]:
                    assert any(r[i] == a and r[j] == b for r in rows), (i, a, j, b)


def test_cases_reach_every_path(hs, eref):
    """the cases take what they are meant to: the zero 4:2:2 chroma macroblock, right-edge slices of 4, 2 and 1 macroblocks, every
    odd height class, both alpha depths with runs below and above 16 and diffs at +-dsize, flat and extreme content, and quantisers past
    max_quant: 16 and above, and the 128 exit"""
    cases = E.all_cases()
    assert any(c.fmt == E.FMT_422 and 1 <= c.w % 16 <= 8 for c in cases)                 # last chroma macroblock at x >= width >> 1
    assert {c.w % 16 for c in cases} >= {0, 1, 2, 9} and any(c.w == 1 for c in cases)
    rests = {((c.w + 15) // 16) % c.mbs_per_slice for c in cases if c.mbs_per_slice == 8}
    assert {r & 4 for r in rests} >= {4} and {r & 2 for r in rests} >= {2} and {r & 1 for r in rests} >= {1}
    assert any(not c.interlaced and c.h % 16 == 1 for c in cases)
    il = [c.h % 32 for c in cases if c.interlaced]
    assert {3, 17, 31} <= set(il)
    for ab in (8, 16):
        runs = [c for c in cases if c.abits == ab and c.alpha == "runs"]
        assert runs
        dsize = 8 if ab == 8 else 64
        a = np.concatenate([c.planes[3].reshape(-1).astype(np.int64) for c in runs])
        coded = a >> 2 if ab == 8 else ((a << 6) | (a >> 4)) & 0xffff
        diffs = np.diff(coded)
        assert (np.abs(diffs) == dsize).any() and (np.abs(diffs) == dsize + 1).any()
        change = np.flatnonzero(diffs != 0)
        lengths = np.diff(change)
        assert (lengths < 16).any() and (lengths > 16).any()
    assert any(c.content == "flat" for c in cases) and any(c.content == "extremes" for c in cases)
    starved = [c for c in E.content_cases() if c.bits_per_mb == 128]
    _, pkts, _, _ = E.run(hs, PU.HostMem(), starved)
    qs = [q for p in pkts for q in E.slice_quants(p)]
    assert any(16 <= q < 128 for q in qs) and 128 in qs


def test_several_frames_one_call(hs, eref):
    """frames of different formats, sizes and options in one call, more than one launch's worth"""
    cases = [c for k, c in enumerate(E.all_cases()) if k % 7 == 0][:11]
    encode_and_compare(hs, eref, cases)


def test_padded_linesizes(hs, eref):
    cases = [E.Case(E.FMT_422, 72, 40, 1, 3, 4, pad=6, seed=500), E.Case(E.FMT_4444, 40, 24, 0, 4, 2, pad=34, seed=501)]
    encode_and_compare(hs, eref, cases)


def test_capacity_one_byte_short(hs, eref):
    """out_capacity one byte short: out_size is -(packet size) and out is untouched; exactly enough: the packet"""
    cases = [E.Case(E.FMT_422, 72, 40, 0, 2, 8, seed=510), E.Case(E.FMT_4444, 56, 34, 2, 4, 4, seed=511)]
    want = [E.ref_encode(eref, c)[0] for c in cases]
    rc, pkts, sizes, raws = E.run(hs, PU.HostMem(), cases, cap_delta=[(len(w), -1) for w in want])
    assert rc == 0
    for w, s, raw in zip(want, sizes, raws):
        assert s == -len(w) and (raw == 0xCD).all()
    rc, pkts, sizes, raws = E.run(hs, PU.HostMem(), cases, cap_delta=[(len(w), 0) for w in want])
    assert rc == 0
    for w, p, raw in zip(want, pkts, raws):
        assert np.array_equal(p, w) and (raw[len(w):] == 0xCD).all()


# ------------------------------------------------------------------------------------------------------------------------------ tables

def test_tables_match_reference(hs, eref):
    """the scans, codebooks, codebook switches, FIRST_DC_CB, quantiser matrices, profile quantiser ranges and bit rates and macroblock
    limits restated in the product are the reference's"""
    a, b = np.zeros(1024, np.int32), np.zeros(1024, np.int32)
    hs.hostsim_prores_enc_tables.restype, hs.hostsim_prores_enc_tables.argtypes = C.c_int, [C.c_void_p]
    n = eref.ref_prores_enc_tables(PU.P(a))
    assert n == 520 and hs.hostsim_prores_enc_tables(PU.P(b)) == n
    assert np.array_equal(a[:n], b[:n]), np.flatnonzero(a[:n] != b[:n])[:8]


# ---------------------------------------------------------------------------------------------------------------------------- refusals

def too_many_slices(w):
    """4096 one-macroblock slices per row over 17 rows"""
    w.width, w.height, w.mbs_per_slice = 65535, 272, 1
    for p in range(4):
        w.linesize[p] = 2 * 65536


def refusals():
    """(name, mutate) pairs, each making the valid work of base_case() one that encode_init or the call refuses"""
    def m(**kw):
        def f(w):
            for k, v in kw.items():
                if isinstance(v, tuple):
                    getattr(w, k)[v[0]] = v[1] if not callable(v[1]) else v[1](getattr(w, k)[v[0]])
                else:
                    setattr(w, k, v)
        return f
    return [
        ("pix_fmt_3", m(pix_fmt=3)), ("pix_fmt_neg", m(pix_fmt=-1)), ("interlaced_3", m(interlaced=3)), ("profile_5", m(profile=5)),
        ("profile_neg", m(profile=-1)), ("mbs_per_slice_3", m(mbs_per_slice=3)), ("mbs_per_slice_0", m(mbs_per_slice=0)),
        ("mbs_per_slice_16", m(mbs_per_slice=16)), ("alpha_bits_4", m(alpha_bits=4)), ("alpha_bits_12", m(alpha_bits=12)),
        ("alpha_bits_32", m(alpha_bits=32)), ("bits_per_mb_1", m(bits_per_mb=1)), ("bits_per_mb_127", m(bits_per_mb=127)),
        ("bits_per_mb_8193", m(bits_per_mb=8193)), ("bits_per_mb_neg", m(bits_per_mb=-1)), ("force_quant_65", m(force_quant=65)),
        ("force_quant_neg", m(force_quant=-1)), ("quant_sel_5", m(quant_sel=5)), ("quant_sel_-2", m(quant_sel=-2)),
        ("vendor_nul", m(vendor=b"ab\x00d")), ("null_y", m(data=(0, None))), ("null_alpha", m(data=(3, None))),
        ("odd_u", m(data=(1, lambda v: v + 1))), ("odd_linesize", m(linesize=(0, lambda v: v + 1))), ("zero_linesize", m(linesize=(2, 0))),
        ("narrow_luma", m(linesize=(0, lambda v: v - 2))), ("narrow_alpha", m(linesize=(3, lambda v: v - 2))),
        ("width_0", m(width=0)), ("height_0", m(height=0)), ("width_65536", m(width=65536)), ("height_65536", m(height=65536)),
        ("too_many_slices", too_many_slices),
        ("interlaced_height_1", m(interlaced=1, height=1)), ("interlaced_height_33", m(interlaced=2, height=33)),
        ("interlaced_height_65", m(interlaced=1, height=65)), ("null_out", m(out=None)), ("null_out_size", m(out_size=None)),
        ("odd_out_size", lambda w: setattr(w, "out_size", w.out_size + 2)),
    ]


def base_case():
    return E.Case(E.FMT_4444, 40, 34, 0, 4, 2, seed=600)


def check_refusals(lib, mem):
    c = base_case()
    ptrs = [mem.put(c.padded(p)) for p in range(4)]
    out = mem.put(np.full(c.capacity(), 0xCD, np.uint8))
    z = mem.put(np.full(2, 0x55, np.int32))
    base = c.work(ptrs, out, c.capacity(), z)
    good = (tables.FFProresEncodeWork * 1)(base)
    need = lib.ff_prores_encode_workspace_cuda(good, 1)
    assert need > 0
    ws = mem.put(np.zeros(need, np.uint8))
    names = []
    for name, mutate in refusals():
        w = tables.FFProresEncodeWork.from_buffer_copy(base)
        mutate(w)
        arr = (tables.FFProresEncodeWork * 2)(tables.FFProresEncodeWork.from_buffer_copy(base), w)   # the valid frame in front is not encoded
        assert lib.ff_prores_encode_workspace_cuda(arr, 2) == 0, name
        lib.avb200_clear_error()
        assert lib.ff_prores_encode_frames_cuda(arr, 2, C.c_void_p(ws), need * 4, None) == -1, name
        assert b"ff_prores_encode_frames_cuda" in (lib.avb200_last_error() or b""), name
        names.append(name)
    for args in ((good, 1, None, need), (good, 1, ws, need - 1), (None, 1, ws, need), (good, -1, ws, need)):
        lib.avb200_clear_error()
        assert lib.ff_prores_encode_frames_cuda(args[0], args[1], None if args[2] is None else C.c_void_p(args[2]), args[3], None) == -1
    lib.avb200_clear_error()
    mem.sync()
    assert (mem.get(out, np.uint8, (c.capacity(),)) == 0xCD).all() and (mem.get(z, np.int32, (2,)) == 0x55).all(), "a refused call wrote"
    assert lib.ff_prores_encode_frames_cuda(good, 0, None, 0, None) == 0
    return names


def test_refusals(hs):
    assert len(check_refusals(hs, PU.HostMem())) == 38


def test_accepted_edges(hs, eref):
    """what encode_init accepts at the edges of the refusals: bits_per_mb 1..127 under force_quant, alpha_bits 12 for a format without
    alpha (not read), interlaced height 2 and 32k + 2, width and height 1"""
    cases = [E.Case(E.FMT_422, 40, 24, 0, 2, 4, bits_per_mb=5, force_quant=3, seed=610),
             E.Case(E.FMT_444, 40, 24, 1, 2, 4, alpha_bits=12, seed=611),
             E.Case(E.FMT_422, 24, 2, 1, 1, 1, seed=612), E.Case(E.FMT_4444, 24, 34, 2, 4, 2, seed=613),
             E.Case(E.FMT_4444, 1, 1, 0, 4, 8, seed=614)]
    encode_and_compare(hs, eref, cases)


def test_workspace_query(hs):
    """the query grows with the frames and sums over a batch; a refused batch or an empty one needs 0 bytes"""
    cs = [E.Case(E.FMT_422, 64, 32, 0, 2, 8, seed=620), E.Case(E.FMT_4444, 128, 64, 1, 4, 2, seed=621)]
    ws = []
    for c in cs:
        arr = (tables.FFProresEncodeWork * 1)(c.work([16] * 4, 16, 1, 16))
        ws.append(hs.ff_prores_encode_workspace_cuda(arr, 1))
    both = (tables.FFProresEncodeWork * 2)(*[c.work([16] * 4, 16, 1, 16) for c in cs])
    assert 0 < ws[0] < ws[1] and hs.ff_prores_encode_workspace_cuda(both, 2) == sum(ws)
    assert hs.ff_prores_encode_workspace_cuda(None, 1) == 0 and hs.ff_prores_encode_workspace_cuda(both, 0) == 0


# ------------------------------------------------------------------------------------------------------------------------- interface

def test_header_exports_and_ctypes_agree(built):
    from libav_b200 import _lib
    hdr = open(os.path.join(ROOT, "include", "avdsp_b200.h")).read()
    names = ["ff_prores_encode_workspace_cuda", "ff_prores_encode_frames_cuda"]
    nm = subprocess.run(["nm", "-D", "--defined-only", _lib.LIB_PATH], capture_output=True, text=True, check=True).stdout
    for n in names:
        assert re.search(r"\b%s\(" % n, hdr), n
        assert re.search(r"\bT %s$" % n, nm, re.M), n
        assert n in _lib.PROTOTYPES, n
    W = tables.FFProresEncodeWork
    exe = os.path.join(hostsim_build.GEN, "prores_enc_abi_probe.%d" % os.getpid())
    os.makedirs(hostsim_build.GEN, exist_ok=True)
    fields = ["data", "linesize", "width", "height", "pix_fmt", "interlaced", "profile", "mbs_per_slice", "bits_per_mb", "quant_sel",
              "alpha_bits", "force_quant", "vendor", "color_primaries", "color_trc", "colorspace", "out", "out_capacity", "out_size"]
    code = '#include <stdio.h>\n#include <stddef.h>\n#include "avdsp_b200.h"\nint main(void){printf("%ld", (long)sizeof(FFProresEncodeWork));' + \
        "".join('printf(" %%ld", (long)offsetof(FFProresEncodeWork, %s));' % f for f in fields) + "return 0;}\n"
    try:
        subprocess.run(["gcc", "-x", "c", "-std=c99", "-I", os.path.join(ROOT, "include"), "-", "-o", exe], input=code, text=True, check=True)
        mine = [int(v) for v in subprocess.run([exe], capture_output=True, text=True, check=True).stdout.split()]
    finally:
        if os.path.exists(exe):
            os.remove(exe)
    assert mine == [C.sizeof(W)] + [getattr(W, f).offset for f in fields]


def test_score_cap_is_unreachable():
    """find_slice_quant's `bits > 65000 * 8` cap cannot fire: the longest codewords the tables allow, for every coefficient of the largest
    slice (8 macroblocks of 4:4:4, |coefficient| <= 32768, so |level| <= 8192 at the smallest quantiser 4) plus 16-bit alpha coded sample by
    sample, stay below it.  So no test can tell the cap from its absence; the product keeps it as the reference has it."""
    def vlc_len(cb, val):
        sb, ro, eo = (cb & 3) + 1, cb >> 5, (cb >> 2) & 7
        sv = sb << ro
        if val >= sv:
            return (val - (sv - (1 << eo))).bit_length() * 2 - 2 - eo + sb + 1
        return (val >> ro) + ro + 1
    coeffs = 8 * 12 * 64
    ac = [0x04, 0x28, 0x4C, 0x05, 0x29, 0x06, 0x0A]
    per_ac = max(vlc_len(cb, coeffs) for cb in ac) + max(vlc_len(cb, 8191) for cb in ac) + 1
    per_dc = max(vlc_len(cb, 2 * 8192 * 2) for cb in [0xB8, 0x04, 0x28, 0x4D, 0x70])
    alpha = 8 * 256 * (16 + 1 + 15)
    assert 3 * 8 * 4 * per_dc + coeffs * per_ac + alpha < 65000 * 8
