"""CPU: MPEG-2 4:2:2 / 4:4:4 pictures and interlaced MPEG-4 pictures through the host-compiled ff_mpv_motion_batch_cuda
(tests/hostsim/), byte for byte against the reference's own ff_mpv_motion over whole padded planes of random bytes; the picture-level
refusals of the new fields, and the records interlaced pictures still reject."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

import hostsim_build
import mpv_ilace_cases as I
import mpv_mc_cases as M

needs_ref = pytest.mark.skipif(not os.path.exists(os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "oracle", "_ref",
                                                               "libmpvcfref.so")), reason="the reference was not built")


@pytest.fixture(scope="session")
def ilsim(built):
    return hostsim_build.fresh()


def check(sim, pics):
    got, rej = I.run_sim(sim, pics)
    want_rej = sum(int((~p.accepted()).sum()) for p in pics)
    assert rej == want_rej
    for g, p in zip(got, pics):
        d = M.first_diff(g, I.run_ref(p))
        assert d is None, d


# ------------------------------------------------------------------------------------------------------------ MPEG-2 4:2:2 and 4:4:4

CF_CASES = [(M.FRAME, 1, 0, 0), (M.FRAME, 1, 0, 1), (M.FRAME, 1, 1, 0), (M.TOP, 1, 0, 0), (M.BOTTOM, 1, 1, 0), (M.TOP, 0, 0, 1),
            (M.BOTTOM, 0, 0, 0)]


@needs_ref
@pytest.mark.parametrize("cf", [2, 3])
@pytest.mark.parametrize("structure,first,b,no_rnd", CF_CASES)
@pytest.mark.parametrize("seed", [1, 2])
def test_chroma_format_matches_reference(ilsim, cf, structure, first, b, no_rnd, seed):
    """every MPEG-2 mv_type of frame and field pictures, first and second fields (the cur reference of a second P field), put / put_no_rnd
    / avg, bi-directional records, vectors at and one step past the skip boundary, far vectors, odd and negative chroma components"""
    rng = np.random.default_rng(1000 * cf + 100 * structure + 10 * seed + 4 * first + 2 * b + no_rnd)
    pic = I.cf_picture(rng, cf, 7, 6, structure=structure, first_field=first, b=b, no_rnd=no_rnd, far=0.15, edge=0.45)
    check(ilsim, [pic])


@needs_ref
def test_chroma_formats_in_one_call(ilsim):
    """4:2:0, 4:2:2 and 4:4:4 MPEG-2 pictures and an interlaced MPEG-4 picture in one call: each kind in launches of its own"""
    rng = np.random.default_rng(77)
    pics = [I.cf_picture(rng, cf, 5, 4, b=1) for cf in (1, 2, 3)] + [I.ilace_picture(rng, 5, 4, qpel=1)]
    check(ilsim, pics)


@needs_ref
@pytest.mark.parametrize("cf", [2, 3])
def test_skip_boundary_exact(ilsim, cf):
    """16X16 vectors one half-sample either side of the skip boundary at every edge: a skipped call leaves chroma as it was too"""
    rng = np.random.default_rng(5 + cf)
    pic = I.CfPicture(rng, cf, 4, 3)
    he, ve = pic.p["h_edge_pos"], pic.p["v_edge_pos"]
    recs = np.zeros(12, M.REC)
    for i, (x, y) in enumerate([(x, y) for y in range(3) for x in range(4)]):
        r = recs[i]
        r["mb_x"], r["mb_y"], r["mv_dir"], r["mv_type"] = x, y, 1, M.T16X16
        edge_x = 2 * (he - 16 - 16 * x)
        edge_y = 2 * (ve - 16 - 16 * y)
        r["mv"][0, 0] = [(edge_x + (i % 3) - 1) if i & 1 else -32 * x - (i % 3) + 1, (edge_y + (i % 3) - 1) if i & 2 else -32 * y - 1 + (i & 1)]
    pic.recs = recs
    check(ilsim, [pic])


# ------------------------------------------------------------------------------------------------------------ interlaced MPEG-4

@needs_ref
@pytest.mark.parametrize("qpel", [0, 1])
@pytest.mark.parametrize("bugs", [0, I.BUG_HPEL_CHROMA, I.BUG_HPEL_CHROMA | M.BUG_QPEL_CHROMA | M.BUG_QPEL_CHROMA2])
@pytest.mark.parametrize("b,no_rnd", [(0, 0), (0, 1), (1, 0)])
@pytest.mark.parametrize("ragged", [0, 1])
def test_interlaced_mpeg4_matches_reference(ilsim, qpel, bugs, b, no_rnd, ragged):
    """FIELD records (half- and quarter-sample, FF_BUG_HPEL_CHROMA on and off, the QPEL_CHROMA bits that must not reach field chroma),
    all four field_select pairs, windows across every edge for both parities, ragged sizes, B-direct field records, mixed with 16X16 and
    8X8"""
    rng = np.random.default_rng(31 * qpel + 7 * bugs + 3 * b + no_rnd + 1000 * ragged)
    pic = I.ilace_picture(rng, 6, 5, b=b, qpel=qpel, bugs=bugs, no_rnd=no_rnd, ragged=bool(ragged), field=0.6, edge=0.5)
    check(ilsim, [pic])


@needs_ref
@pytest.mark.parametrize("qpel", [0, 1])
@pytest.mark.parametrize("fs", [(0, 0), (0, 1), (1, 0), (1, 1)])
def test_field_windows_across_edges(ilsim, qpel, fs):
    """every macroblock a FIELD record whose both fields sit just across the top or bottom edge of the field: the emulated window is
    clamped in frame rows, so edge rows come from the other parity"""
    rng = np.random.default_rng(11 + 2 * fs[0] + fs[1] + 10 * qpel)
    pic = I.IlacePicture(rng, 3, 3, qpel=qpel, width=44, height=42)
    unit = 4 if qpel else 2
    vh = pic.p["v_edge_pos"] // 2
    recs = np.zeros(9, I.G.REC)
    for i in range(9):
        x, y = i % 3, i // 3
        r = recs[i]
        r["mb_x"], r["mb_y"], r["mv_dir"], r["mv_type"] = x, y, 1, M.TFIELD
        r["field_select"][0] = fs
        for f in range(2):
            top = (i + f) & 1
            t = (-1 - (i % 4)) if top else vh - 8 + 1 + (i % 4)
            r["mv"][0, f] = [unit * ((i % 5) - 2) + (i & (unit - 1)), unit * (t - 8 * y) + ((i + f) % unit)]
    pic.recs = recs
    check(ilsim, [pic])


@needs_ref
@pytest.mark.parametrize("qpel", [0, 1])
def test_interlaced_svop(ilsim, qpel):
    """an interlaced S-VOP: mcsel 16X16 records through GMC, FIELD and 8X8 records through the plain body"""
    rng = np.random.default_rng(400 + qpel)
    pic = I.ilace_picture(rng, 6, 5, qpel=qpel, sprite=True, field=0.4)
    assert (pic.recs["mv_type"] == M.TFIELD).any() and pic.recs["mcsel"].any()
    check(ilsim, [pic])


@needs_ref
def test_interlaced_rejects_16x8_and_dmv(ilsim):
    """16X8 and DMV records stay outside the H.263 family in interlaced pictures: counted, their macroblocks untouched"""
    rng = np.random.default_rng(9)
    pic = I.ilace_picture(rng, 5, 4, b=1)
    pic.recs["mv_type"][::4] = M.T16X8
    pic.recs["mv_type"][1::4] = M.TDMV
    assert (~pic.accepted()).sum() >= 8
    check(ilsim, [pic])


@needs_ref
def test_interlaced_flag_ignored_in_mpeg2(ilsim):
    """interlaced is read in out_format 2 pictures only: an MPEG-2 picture with it set reconstructs as without it"""
    rng = np.random.default_rng(12)
    pic = I.cf_picture(rng, 2, 5, 4)
    pic.interlaced = 1
    check(ilsim, [pic])


# ------------------------------------------------------------------------------------------------------------ refusals and layout

def _refused(sim, pic, **fields):
    frame = [a.copy() for a in pic.frame]
    recs = np.ascontiguousarray(pic.recs)
    base = [a.ctypes.data for a in frame]
    s = I.set_fields(M.picture_struct(pic, base, base, [a.ctypes.data for a in pic.last], [a.ctypes.data for a in pic.next],
                                      recs.ctypes.data, len(recs)), pic)
    for k, v in fields.items():
        setattr(s, k, v)
    rej = np.zeros(1, np.uint32)
    sim.avb200_clear_error()
    rc = sim.ff_mpv_motion_batch_cuda(C.byref(s), 1, rej.ctypes.data, None)
    unchanged = all(np.array_equal(a, b) for a, b in zip(frame, pic.frame)) and rej[0] == 0
    return rc, sim.avb200_last_error(), unchanged


@pytest.mark.parametrize("fmt,cf", [(2, 2), (2, 3), (0, 0), (0, 4), (2, 0), (2, 4), (0, -1)])
def test_chroma_format_refusals(ilsim, fmt, cf):
    rng = np.random.default_rng(3)
    pic = I.ilace_picture(rng, 4, 3) if fmt == 2 else I.cf_picture(rng, 3, 4, 3)
    rc, err, unchanged = _refused(ilsim, pic, chroma_format=cf)
    assert rc == -1 and b"chroma_format" in err and unchanged


def test_interlaced_obmc_refused(ilsim):
    """interlaced with OBMC in a P picture is refused (H.263 has no interlace); in a B picture obmc is ignored, as in C"""
    rng = np.random.default_rng(4)
    pic = I.ilace_picture(rng, 4, 3)
    obmc = np.zeros(len(pic.recs), np.dtype([("b", "u1", (44,))]))        # FFMpvOBMCRecord storage: never read, the call is refused
    rc, err, unchanged = _refused(ilsim, pic, obmc=1, obmc_recs=obmc.ctypes.data)
    assert rc == -1 and b"interlaced" in err and unchanged
    b = I.ilace_picture(rng, 4, 3, b=1)
    rc, err, _ = _refused(ilsim, b, obmc=1)
    assert rc == 0, err


def test_uvlinesize_checked_against_chroma_width(ilsim):
    """a 4:4:4 picture's uvlinesize must exceed 16 * mb_width, not 8 * mb_width"""
    rng = np.random.default_rng(6)
    pic = I.cf_picture(rng, 3, 4, 3)
    rc, err, unchanged = _refused(ilsim, pic, uvlinesize=8 * 4 + 1, pic_uvlinesize=8 * 4 + 1)
    assert rc == -1 and b"uvlinesize" in err and unchanged


def test_header_layout(built, tmp_path):
    """include/avdsp_b200.h as C compiles it: interlaced ends FFMpvMCPicture where libav_b200/tables.py puts it"""
    from libav_b200 import tables
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    src = tmp_path / "probe.c"
    src.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "avdsp_b200.h"\nint main(void) { printf("%d %d", '
                   '(int)sizeof(FFMpvMCPicture), (int)offsetof(FFMpvMCPicture, interlaced)); return 0; }\n')
    exe = str(tmp_path / "probe")
    subprocess.check_call(["gcc", "-std=c99", "-Wall", "-Werror", "-I", os.path.join(root, "include"), str(src), "-o", exe])
    P = tables.FFMpvMCPicture
    assert [int(x) for x in subprocess.check_output([exe]).split()] == [C.sizeof(P), P.interlaced.offset]
