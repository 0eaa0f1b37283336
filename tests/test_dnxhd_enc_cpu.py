"""The VC-3 / DNxHD encoder (libav_b200/csrc/dnxhd_enc.cu + dnxhd_enc.cuh) compiled as host C++ (tests/hostsim/dnxhd_enc_hostsim.cpp) against
the reference encoder (oracle/_ref/libdnxhdencref.so: dnxhdenc.c, unmodified): whole packets byte for byte, out_info and the rate-control
state after every frame, over every CID, both rate controls, both field orders, the three forward DCTs, qmax and nitris_compat, content
that takes every path of the rate controls, sequences through one state, linesizes and the lines under 10-bit 1080-line pictures.  Also
the VLC tables built from each CID, the CIDEntry layout, header / exports / ctypes agreement and every refusal."""
import ctypes as C
import os
import re
import subprocess

import numpy as np
import pytest

import hostsim_build
import prores_util as PU
import dnxhd_enc_util as E
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
    lib = hostsim_build.load()
    lib.hostsim_dnxhd_vlc.restype = C.c_int
    lib.hostsim_dnxhd_vlc.argtypes = [C.c_void_p] * 5
    return lib


def cid_cases():
    """every CID, fast and RD alternating; the interlaced CIDs in both field orders and both rate controls; 8-bit CIDs through islow,
    ifast and FAAN in turn"""
    cs = []
    for k, cid in enumerate(E.CIDS):
        dct = 0 if cid in E.TEN_BIT else (0, E.FASTINT, E.FAAN)[k % 3]
        cs.append(E.Case(cid, ["natural"], dct_algo=dct, mb_decision=E.RD if k % 2 else 0, qmax=31 if k % 2 == 0 else 12, seed=10 + k))
    for k, cid in enumerate(E.INTERLACED):
        dct = 0 if cid in E.TEN_BIT else (E.FAAN, E.FASTINT)[k % 2]
        cs.append(E.Case(cid, ["natural"], interlaced=2, dct_algo=dct, mb_decision=0 if k % 2 else E.RD, qmax=10, seed=30 + k))
    return cs


def option_cases():
    """qmax 2 / 3 / 31 / 69 and nitris_compat 0 / 1, at both depths and with both rate controls"""
    return [E.Case(1251, ["natural"], qmax=2, seed=40), E.Case(1250, ["natural"], qmax=3, mb_decision=E.RD, seed=41),
            E.Case(1258, ["noise"], qmax=69, seed=42), E.Case(1252, ["natural"], qmax=69, mb_decision=E.RD, nitris=1, seed=43),
            E.Case(1251, ["noise"], qmax=31, nitris=1, seed=44), E.Case(1250, ["noise"], qmax=31, nitris=1, seed=45)]


def content_cases():
    """flat frames (qscale 1 fits: no variance pass), gradients (variance ties), noise (the lambda and qscale searches upwards), 0 / max
    checkerboards (a rate-control failure at a small qmax, and with RD)"""
    return [E.Case(1251, ["flat", "flat"], seed=50), E.Case(1250, ["gradient"], seed=51), E.Case(1258, ["gradient"], dct_algo=E.FASTINT, seed=52),
            E.Case(1252, ["noise"], mb_decision=E.RD, qmax=8, seed=53), E.Case(1258, ["checker"], qmax=3, seed=54),
            E.Case(1250, ["checker"], qmax=3, mb_decision=E.RD, seed=55), E.Case(1251, ["checker"], seed=56)]


def sequence_cases():
    """4-8 frames through one state: the searches start where the last field left the state, both directions of the lambda search, and a
    rate-control failure followed by a frame that fits (the post-failure state is compared with the reference's)"""
    return [E.Case(1251, ["natural", "noise", "flat", "natural", "gradient"], seed=60),
            E.Case(1250, ["noise", "natural", "flat", "noise"], mb_decision=E.RD, qmax=10, seed=61),
            E.Case(1258, ["natural", "checker", "flat", "checker", "natural", "noise"], qmax=3, seed=62),
            E.Case(1252, ["flat", "checker", "natural", "noise"], qmax=3, mb_decision=E.RD, seed=63),
            E.Case(1260, ["natural", "noise", "natural", "flat"], interlaced=2, qmax=12, seed=64),
            E.Case(1243, ["fields", "natural", "fields"], interlaced=1, qmax=12, seed=65),
            E.Case(1242, ["fields", "natural"], interlaced=1, qmax=12, mb_decision=E.RD, seed=66)]


def layout_cases():
    """padded linesizes, odd 8-bit linesizes, and seeded lines under a 10-bit 1080-line picture"""
    return [E.Case(1251, ["natural"], pad=96, seed=70), E.Case(1258, ["natural", "noise"], odd=True, seed=71),
            E.Case(1242, ["natural"], odd=True, interlaced=2, qmax=8, seed=72), E.Case(1235, ["natural"], pad=64, tails=[5], qmax=8, seed=73),
            E.Case(1241, ["natural"], pad=2, tails=[6], qmax=8, seed=74)]


GROUPS = {"cids": cid_cases, "options": option_cases, "content": content_cases, "sequences": sequence_cases, "layout": layout_cases}


@pytest.mark.parametrize("group", sorted(GROUPS))
def test_packets_match_reference_encoder(hs, eref, group):
    """every case of the group in one call, each through its own state; packets, out_info and the final state equal the reference's"""
    E.check(hs, eref, PU.HostMem(), GROUPS[group]())


@pytest.mark.parametrize("k", range(len(sequence_cases())))
def test_state_after_every_frame(hs, eref, k):
    """each sequence one frame per call through one state: qscale and lambda after every frame, a failed one included, are the reference
    context's (a field continues from the state the previous field left)"""
    E.check_states(hs, eref, PU.HostMem(), sequence_cases()[k])


def test_groups_reach_every_path(eref):
    """the reference takes the paths the cases are there for: a failure, a frame that fits after one, qscale 1 fitting, qscale 2+"""
    seen = set()
    for c in content_cases() + sequence_cases():
        _, rc = E.ref_encode(eref, c)
        for k in range(len(rc)):
            if rc[k, 0] < 0:
                seen.add("fail")
                if k + 1 < len(rc) and rc[k + 1, 0] >= 0:
                    seen.add("fit after fail")
            elif c.mb_decision != E.RD:
                seen.add("qscale 1" if rc[k, 1] == 1 else "qscale > 1")
    assert seen == {"fail", "fit after fail", "qscale 1", "qscale > 1"}, seen


def test_several_states_in_one_call(hs, eref):
    """frames of several states interleaved in one call: each state's frames in array order, the states independent"""
    cases = [E.Case(1251, ["natural", "noise"], seed=80), E.Case(1258, ["noise", "flat"], mb_decision=E.RD, qmax=6, seed=81),
             E.Case(1250, ["gradient"], seed=82)]
    E.check(hs, eref, PU.HostMem(), cases)


def test_padding_lines_under_10bit_1080(hs, eref):
    """the 8 lines under a 10-bit 1080-line picture: another seed changes the product's packet exactly when it changes the reference's"""
    a = E.Case(1235, ["natural"], tails=[1], qmax=31, seed=90)
    b = E.Case(1235, ["natural"], tails=[2], qmax=31, seed=90)
    pa, _ = E.check(hs, eref, PU.HostMem(), [a])
    pb, _ = E.check(hs, eref, PU.HostMem(), [b])
    wa, _ = E.ref_encode(eref, a)
    wb, _ = E.ref_encode(eref, b)
    assert (not np.array_equal(pa[0], pb[0])) == (not np.array_equal(wa[0], wb[0]))


def test_ibias_does_not_reach_the_packet(eref):
    """the encoder's ibias option only reaches qmatrix_*16, which ff_dct_quantize_c never reads: the reference's packets do not change"""
    base = None
    for ibias in (999999, 0, -200, 300, 1 << 20):
        c = E.Case(1238, ["natural"], ibias=ibias, seed=95)
        pk, rc = E.ref_encode(eref, c)
        if base is None:
            base = pk[0]
        assert np.array_equal(pk[0], base), ibias


@pytest.mark.parametrize("cid", E.CIDS)
def test_vlc_tables_match_reference(hs, eref, cid):
    """dnxhd_init_vlc's vlc / run tables, built by the product from the CID entry"""
    n = 4 * 4096
    got = [np.zeros(n, np.uint32), np.zeros(n, np.uint8), np.zeros(63, np.uint16), np.zeros(63, np.uint8)]
    want = [np.zeros(n, np.uint32), np.zeros(n, np.uint8), np.zeros(63, np.uint16), np.zeros(63, np.uint8)]
    ml = eref.ref_dnxhd_vlc(C.byref(E.Case.__new__(E.Case).opts.__func__(type("O", (), dict(
        cid=cid, interlaced=0, dct_algo=0, mb_decision=0, qmax=31, nitris=0, ibias=999999))())), *[PU.P(a) for a in want])
    assert ml == hs.hostsim_dnxhd_vlc(eref.ref_dnxhd_cid_entry(cid), *[PU.P(a) for a in got])
    for g, w, m in zip(got, want, (4 * ml, 4 * ml, 63, 63)):
        assert np.array_equal(g[:m], w[:m])


def test_cid_entry_layout(eref):
    """FFDnxhdCidEntry (and its ctypes mirror) has CIDEntry's size and field offsets"""
    out = np.zeros(32, np.int32)
    n = eref.ref_dnxhd_cid_layout(PU.P(out))
    S = tables.FFDnxhdCidEntry
    assert out[0] == C.sizeof(S)
    assert list(out[1:n]) == [getattr(S, f).offset for f, _ in S._fields_]
    e = C.cast(eref.ref_dnxhd_cid_entry(1243), C.POINTER(S))[0]
    assert (e.cid, e.width, e.height, e.interlaced, e.bit_depth) == (1243, 1920, 1080, 1, 8)


def test_header_exports_and_ctypes_agree(built):
    """the public header declares both calls and the three structs; the library exports the calls; _lib has their prototypes; the
    ctypes structs have the header's fields in order"""
    hdr = open(os.path.join(ROOT, "include", "avdsp_b200.h")).read()
    from libav_b200 import _lib
    syms = subprocess.run(["nm", "-D", "--defined-only", os.path.join(ROOT, "libav_b200", "libavdsp_b200.so")], capture_output=True,
                          text=True).stdout
    for f in ("ff_dnxhd_encode_workspace_cuda", "ff_dnxhd_encode_frames_cuda"):
        assert re.search(r"\b%s\(" % f, hdr) and f in _lib.PROTOTYPES and re.search(r" T %s$" % f, syms, re.M), f
    for name, fields in (("FFDnxhdEncodeWork", ["data", "linesize", "cid_table", "interlaced", "dct_algo", "mb_decision", "qmax",
                                                "nitris_compat", "state", "out", "out_capacity", "out_info"]),
                         ("FFDnxhdRcState", ["qscale", "lambda_"])):
        assert [f for f, _ in getattr(tables, name)._fields_] == fields
        body = re.search(r"typedef struct %s \{(.*?)\} %s;" % (name, name), hdr, re.S).group(1)
        decl = re.sub(r"/\*.*?\*/", "", body, flags=re.S)
        names = re.findall(r"\**(\w+)(?:\[\d+\])?\s*[,;]", decl)
        assert names == [f.rstrip("_") for f in fields], (name, names)


def refusal_cases(eref):
    """(description, work mutator, workspace delta) for each refusal"""
    bad_runs = (C.c_uint8 * 62)(*([0] + list(range(2, 63))))
    dup_runs = (C.c_uint8 * 62)(*([1, 1] + list(range(3, 63))))
    no_level = (C.c_uint8 * 257)(*([0] * 257))

    def entry(**kw):
        e = tables.FFDnxhdCidEntry.from_buffer_copy(C.cast(eref.ref_dnxhd_cid_entry(1251), C.POINTER(tables.FFDnxhdCidEntry))[0])
        for k, v in kw.items():
            setattr(e, k, v)
        entry.keep.append(e)
        return C.addressof(e)
    entry.keep = [bad_runs, dup_runs, no_level]
    other = eref.ref_dnxhd_cid_entry(1243)
    return [
        ("NULL plane", lambda w: setattr(w, "data", (C.c_void_p * 3)(0, w.data[1], w.data[2]))),
        ("narrow luma linesize", lambda w: w.linesize.__setitem__(0, 1279)),
        ("narrow chroma linesize", lambda w: w.linesize.__setitem__(2, 639)),
        ("zero linesize", lambda w: w.linesize.__setitem__(1, 0)),
        ("NULL cid_table", lambda w: setattr(w, "cid_table", None)),
        ("interlacing mismatch", lambda w: setattr(w, "interlaced", 1)),
        ("interlaced CID as progressive", lambda w: (setattr(w, "cid_table", other), setattr(w, "interlaced", 0))),
        ("interlaced 3", lambda w: setattr(w, "interlaced", 3)),
        ("bit depth 9", lambda w: setattr(w, "cid_table", entry(bit_depth=9))),
        ("run of 0", lambda w: setattr(w, "cid_table", entry(run=C.addressof(bad_runs)))),
        ("run listed twice", lambda w: setattr(w, "cid_table", entry(run=C.addressof(dup_runs)))),
        ("level without code", lambda w: setattr(w, "cid_table", entry(ac_level=C.addressof(no_level)))),
        ("qmax 1", lambda w: setattr(w, "qmax", 1)),
        ("qmax 70", lambda w: setattr(w, "qmax", 70)),
        ("nitris 2", lambda w: setattr(w, "nitris_compat", 2)),
        ("capacity one byte short", lambda w: setattr(w, "out_capacity", w.out_capacity - 1)),
        ("NULL out", lambda w: setattr(w, "out", None)),
        ("misaligned out", lambda w: setattr(w, "out", w.out + 2)),
        ("NULL state", lambda w: setattr(w, "state", None)),
        ("NULL out_info", lambda w: setattr(w, "out_info", None)),
    ]


def check_refusals(lib, eref, mem):
    """each refusal in a batch after a good frame: -1, a message, and nothing launched (the good frame's out_info stays untouched); then a
    workspace one byte short; then 10-bit odd linesizes and planes"""
    good = E.Case(1251, ["flat"], seed=99)
    for name, mut in refusal_cases(eref):
        works = []
        for c in (good, good):
            planes, lss = c.frames[0]
            w = tables.FFDnxhdEncodeWork()
            for p in range(3):
                w.data[p] = mem.put(planes[p]); w.linesize[p] = lss[p]
            w.cid_table = eref.ref_dnxhd_cid_entry(1251)
            w.qmax = 31
            w.state = mem.put(np.array([1, 2048], np.uint32))
            w.out = mem.put(np.zeros(458752, np.uint8)); w.out_capacity = 458752
            w.out_info = mem.put(np.full(2, 7, np.int32))
            works.append(w)
        mut(works[1])
        arr = (tables.FFDnxhdEncodeWork * 2)(*works)
        ws = mem.put(np.zeros(1 << 26, np.uint8))
        lib.avb200_clear_error()
        assert lib.ff_dnxhd_encode_frames_cuda(arr, 2, C.c_void_p(ws), 1 << 26, None) == -1, name
        assert lib.avb200_last_error(), name
        lib.avb200_clear_error()
        mem.sync()
        assert list(mem.get(works[0].out_info, np.int32, (2,))) == [7, 7], name
    rc, *_ = E.run(lib, eref, mem, [good], ws_delta=-1)
    assert rc == -1 and lib.avb200_last_error()
    lib.avb200_clear_error()
    ten = E.Case(1250, ["flat"], seed=98)
    for p in range(3):
        for what in ("linesize", "data"):
            planes, lss = ten.frames[0]
            w = tables.FFDnxhdEncodeWork()
            for q in range(3):
                w.data[q] = mem.put(planes[q]); w.linesize[q] = lss[q]
            if what == "linesize":
                w.linesize[p] += 1
            else:
                w.data[p] += 1
            w.cid_table = eref.ref_dnxhd_cid_entry(1250)
            w.qmax, w.state = 31, mem.put(np.array([1, 2048], np.uint32))
            w.out, w.out_capacity, w.out_info = mem.put(np.zeros(458752, np.uint8)), 458752, mem.put(np.zeros(2, np.int32))
            arr = (tables.FFDnxhdEncodeWork * 1)(w)
            assert lib.ff_dnxhd_encode_workspace_cuda(arr, 1) == 0
            assert lib.ff_dnxhd_encode_frames_cuda(arr, 1, C.c_void_p(mem.put(np.zeros(1 << 26, np.uint8))), 1 << 26, None) == -1
            lib.avb200_clear_error()


def test_refusals(hs, eref):
    check_refusals(hs, eref, PU.HostMem())
