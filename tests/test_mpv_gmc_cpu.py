"""CPU: MPEG-4 global motion compensation (S-VOPs) in ff_mpv_motion_batch_cuda and the MpegVideoDSPContext slots.  The product
(libav_b200/csrc/mpv_gmc.cuh through mpv_mc.cu, compiled for the host by tests/hostsim/mpv_mc_hostsim.cpp; the slots of mpegvideodsp.cu
through tests/hostsim/mpegvideodsp_hostsim.cpp) and the plain-C port (oracle/port/orc_mpvgmc.c) against the reference's real
ff_mpv_motion on S-VOPs and its gmc1_c / ff_gmc_c (oracle/_ref/libmpvgmcref.so, libavref.so): 1, 2 and 3 warping points at every
accuracy, both roundings; mcsel 16X16, plain half- and quarter-sample 16X16, 4MV with mcsel left set, intra macroblocks; ragged and tiny
pictures; hand-set parameters on every side of the picture; the slots at every fraction; the table layout; the refusals."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

import hostsim_build
import mpv_gmc_cases as G
import mpv_mc_cases as M


@pytest.fixture(scope="module")
def gref(built):
    lib = G.ref_lib()
    if lib is None:
        pytest.skip("oracle/_ref not built (no reference tree in this environment)")
    return lib


@pytest.fixture
def gsim(built):
    return hostsim_build.fresh()


@pytest.fixture(scope="module")
def gport(built):
    return G.port_lib()


CASES = [(pts, acc, no_rnd, qpel) for pts in (1, 2, 3) for acc in range(4) for no_rnd in (0, 1) for qpel in (0, 1)]


def _svop(seed, mb_w, mb_h, pts, acc, no_rnd, qpel, ragged=True):
    rng = np.random.default_rng(seed)
    pic = G.svop(rng, mb_w, mb_h, params=(0, 1, [[0, 0], [0, 0]], [[2, 0], [0, 2]]), no_rnd=no_rnd, qpel=qpel, ragged=ragged)
    p = pic.p
    pic.sprite = G.random_params(rng, p["width"], p["height"], mb_w, mb_h, p["h_edge_pos"], p["v_edge_pos"], pts=pts, acc=acc)
    return pic


@pytest.mark.parametrize("pts,acc,no_rnd,qpel", CASES)
def test_hostsim_matches_reference(gref, gsim, pts, acc, no_rnd, qpel):
    for seed in range(2):
        pic = _svop(1000 * pts + 100 * acc + 10 * no_rnd + qpel + 7 * seed, 7, 5, pts, acc, no_rnd, qpel, ragged=bool(seed))
        assert pic.sprite[1] == pts or pts > 1      # a random 2- / 3-point warp is never a translation in practice
        got, rej = G.run_sim(gsim, [pic])
        assert rej == 0
        d = M.first_diff(got[0], G.run_ref(gref, pic))
        assert d is None, (seed, pic.sprite, d)


@pytest.mark.parametrize("pts,acc,no_rnd,qpel", CASES)
def test_port_matches_reference(gref, gport, pts, acc, no_rnd, qpel):
    for seed in range(2):
        pic = _svop(5000 + 1000 * pts + 100 * acc + 10 * no_rnd + qpel + 7 * seed, 7, 5, pts, acc, no_rnd, qpel, ragged=bool(seed))
        d = M.first_diff(G.run_ref(gport, pic), G.run_ref(gref, pic))
        assert d is None, (seed, pic.sprite, d)


def test_trajectories_reduce_translations():
    """a warp whose displacements move every reference point alike is a translation: reduced to one point, delta a"""
    for acc in range(4):
        for n in (2, 3):
            d = np.array([[5, -3], [0, 0], [0, 0]])
            p = G.trajectory(352, 288, acc, n, d)
            assert p is not None and p[1] == 1 and p[3] == [[2 << acc, 0], [0, 2 << acc]], (acc, n, p)
        assert G.trajectory(352, 288, acc, 0, np.zeros((3, 2), int))[1] == 1


@pytest.mark.parametrize("kind", ["clamp", "edge1", "hpel1"])
def test_raw_parameters(gref, gsim, gport, kind):
    """hand-set parameters: positions on every side of and wholly outside the picture, gmc1 clipped to width / height, whole / half-sample
    gmc1 offsets -- both roundings, ragged and tiny pictures (h_edge_pos below 17 included)"""
    for seed in range(24):
        rng = np.random.default_rng(300 + seed)
        mb_w, mb_h = (int(rng.integers(1, 3)), int(rng.integers(1, 3))) if seed % 3 == 0 else (5, 4)
        pic = G.svop(rng, mb_w, mb_h, params=(0, 1, [[0, 0], [0, 0]], [[2, 0], [0, 2]]), no_rnd=seed & 1, qpel=(seed >> 1) & 1,
                     ragged=seed % 2 == 0, mcsel=0.85, intra=0.05)
        pic.sprite = G.raw_params(rng, pic, kind, int(rng.integers(0, 4)))
        want = G.run_ref(gref, pic)
        got, rej = G.run_sim(gsim, [pic])
        assert rej == 0 and M.first_diff(got[0], want) is None, (seed, pic.sprite, M.first_diff(got[0], want))
        assert M.first_diff(G.run_ref(gport, pic), want) is None, (seed, pic.sprite)


def test_clamp_branches_are_reached():
    """the 'clamp' parameter sets place samples in each of ff_gmc_c's four branches (a picture's luma positions, counted in Python)"""
    hit = set()
    for seed in range(24):
        rng = np.random.default_rng(300 + seed)
        mb_w, mb_h = (int(rng.integers(1, 3)), int(rng.integers(1, 3))) if seed % 3 == 0 else (5, 4)
        pic = G.svop(rng, mb_w, mb_h, params=(0, 1, [[0, 0], [0, 0]], [[2, 0], [0, 2]]), no_rnd=seed & 1, qpel=(seed >> 1) & 1,
                     ragged=seed % 2 == 0, mcsel=0.85, intra=0.05)
        acc, pts, off, d = G.raw_params(rng, pic, "clamp", int(rng.integers(0, 4)))
        W, H, sh = pic.p["h_edge_pos"] - 1, pic.p["v_edge_pos"] - 1, 16 + acc + 1
        for y in range(0, 16 * mb_h, 3):
            for x in range(0, 16 * mb_w, 3):
                sx, sy = (off[0][0] + d[0][0] * x + d[0][1] * y) >> sh, (off[0][1] + d[1][0] * x + d[1][1] * y) >> sh
                hit.add((0 <= sx < W, 0 <= sy < H))
    assert hit == {(True, True), (True, False), (False, True), (False, False)}


def test_stacked_and_mixed_call(gref, gsim):
    """S-VOPs with P and B pictures in one call, more than one launch of S-VOPs; each picture as the reference computes it"""
    pics = []
    for i in range(18):
        pics.append(_svop(40 + i, 3, 3, 1 + i % 3, i % 4, i & 1, (i >> 1) & 1))
    rng = np.random.default_rng(90)
    for b in (0, 1):
        p = M.Picture(rng, 2, 3, 3, b=b, qpel=1)
        M.make_records(rng, p)
        pics.append(p)
    got, rej = G.run_sim(gsim, pics)
    assert rej == 0
    for i, p in enumerate(pics):
        assert M.first_diff(got[i], G.run_ref(gref, p)) is None, i


def test_rejected_records_count(gsim):
    """records the kernel cannot take leave their macroblock untouched and are counted, as in plain pictures"""
    pic = _svop(77, 4, 3, 2, 1, 0, 0)
    pic.recs["mb_x"][:2] = 200
    pic.recs["mv_type"][2] = M.TFIELD
    got, rej = G.run_sim(gsim, [pic])
    assert rej == 3


# ------------------------------------------------------------------------------------------------------------------------------- refusals

REFUSALS = [("b_picture", 1), ("obmc", 1), ("picture_structure", 1), ("out_format", 0), ("real_sprite_warping_points", 0),
            ("real_sprite_warping_points", 4), ("sprite_warping_accuracy", -1), ("sprite_warping_accuracy", 4)]


@pytest.mark.parametrize("field,value", REFUSALS)
def test_refusals_change_nothing(gsim, field, value):
    pic = _svop(3, 4, 4, 2, 2, 0, 0, ragged=False)
    frame = [a.copy() for a in pic.frame]
    recs = np.ascontiguousarray(pic.recs)
    arr = G.structs([pic], [[a.ctypes.data for a in frame]], [recs])
    setattr(arr[0], field, value)
    if field == "obmc":
        arr[0].obmc_recs = recs.ctypes.data
    if field == "picture_structure":
        arr[0].pic_linesize, arr[0].pic_uvlinesize = 2 * arr[0].linesize, 2 * arr[0].uvlinesize
    rej = np.zeros(1, np.uint32)
    assert gsim.ff_mpv_motion_batch_cuda(C.cast(arr, C.c_void_p), 1, rej.ctypes.data, None) == -1
    assert b"sprite" in gsim.avb200_last_error()
    assert all(np.array_equal(a, b) for a, b in zip(frame, pic.frame)) and rej[0] == 0


def test_zeroed_sprite_picture_is_refused(gsim):
    """sprite set with every sprite field zero (what a caller unaware of GMC sends) is still refused"""
    pic = _svop(4, 3, 3, 1, 0, 0, 0)
    frame = [a.copy() for a in pic.frame]
    recs = np.ascontiguousarray(pic.recs)
    arr = G.structs([pic], [[a.ctypes.data for a in frame]], [recs])
    arr[0].sprite_warping_accuracy = arr[0].real_sprite_warping_points = 0
    for i in range(2):
        for k in range(2):
            arr[0].sprite_offset[i][k] = arr[0].sprite_delta[i][k] = 0
    rej = np.zeros(1, np.uint32)
    assert gsim.ff_mpv_motion_batch_cuda(C.cast(arr, C.c_void_p), 1, rej.ctypes.data, None) == -1
    assert b"sprite" in gsim.avb200_last_error()
    assert all(np.array_equal(a, b) for a, b in zip(frame, pic.frame)) and rej[0] == 0


# ------------------------------------------------------------------------------------------------------------------------------- slots

def _slot_tables(lib_init, ref):
    from libav_b200 import tables
    ours, theirs = tables.MpegVideoDSPContext(), tables.MpegVideoDSPContext()
    lib_init(C.byref(ours))
    ref.ref_mpegvideodsp_init(C.byref(theirs))
    return ours, theirs


def _plane(rng, w, h, stride):
    return rng.integers(0, 256, (h, stride), dtype=np.uint8)


def test_slots_gmc1_match_reference(gref, gsim):
    """gmc1 for every (x16, y16), rounder 127 / 128, h 8 / 16: the slot's kernel and staging against gmc1_c"""
    ours, theirs = _slot_tables(gsim.ff_mpegvideodsp_init_cuda, gref)
    rng = np.random.default_rng(11)
    stride = 40
    for h in (8, 16):
        src = _plane(rng, 24, h + 4, stride)
        for x16 in range(16):
            for y16 in range(16):
                for rounder in (127, 128):
                    dst0 = _plane(rng, 24, h + 2, stride)
                    dst1 = dst0.copy()
                    sp = src.ctypes.data + stride + 3
                    ours.gmc1(C.cast(dst0.ctypes.data + 2, C.POINTER(C.c_uint8)), C.cast(sp, C.POINTER(C.c_uint8)), stride, h, x16, y16, rounder)
                    theirs.gmc1(C.cast(dst1.ctypes.data + 2, C.POINTER(C.c_uint8)), C.cast(sp, C.POINTER(C.c_uint8)), stride, h, x16, y16, rounder)
                    assert np.array_equal(dst0, dst1), (h, x16, y16, rounder)


def test_slots_gmc_match_reference(gref, gsim, gport):
    """gmc at shift 1..4 with random r, positions inside, across and outside the plane (every branch), near-identity and skewed maps, and
    maps whose corners leave int32 (the whole plane staged); against ff_gmc_c and the port"""
    ours, theirs = _slot_tables(gsim.ff_mpegvideodsp_init_cuda, gref)
    rng = np.random.default_rng(12)
    u8 = lambda a, o=0: C.cast(a.ctypes.data + o, C.POINTER(C.c_uint8))
    for it in range(1500):
        shift = 1 + it % 4
        h = (8, 16)[(it >> 2) & 1]
        w, hh = int(rng.integers(2, 48)), int(rng.integers(2, 40))
        stride = max(w, 8) + int(rng.integers(0, 9))          # the 8 x h destination shares the stride
        src = _plane(rng, w, max(hh, h), stride)
        one = 1 << (16 + shift)
        x, y = int(rng.integers(-20, w + 20)), int(rng.integers(-20, hh + 20))
        ox, oy = x * one + int(rng.integers(0, one)), y * one + int(rng.integers(0, one))
        dxx, dyy = int(one * rng.uniform(0.3, 1.7)), int(one * rng.uniform(0.3, 1.7))
        dxy, dyx = int(one * rng.uniform(-0.6, 0.6)), int(one * rng.uniform(-0.6, 0.6))
        if it % 50 == 0:                 # a corner beyond int32: C's sums wrap (gcc), the slot stages the whole plane
            ox = int(np.int32(2 ** 31 - 1 - int(rng.integers(0, 4 * abs(dxx) + 1))))
        if not all(G._fits(ox + dxx * cx + dxy * cy, oy + dyx * cx + dyy * cy) for cx in (0, 8) for cy in (0, h)) and it % 50:
            continue
        r = int(rng.integers(0, 1 << (2 * shift)))
        dst = [rng.integers(0, 256, (h, stride), dtype=np.uint8) for _ in range(3)]
        dst[1][:] = dst[2][:] = dst[0]
        args = (stride, h, ox, oy, dxx, dxy, dyx, dyy, shift, r, w, hh)
        ours.gmc(u8(dst[0]), u8(src), *args)
        theirs.gmc(u8(dst[1]), u8(src), *args)
        gport.gmc(dst[2].ctypes.data, src.ctypes.data, *args)
        assert np.array_equal(dst[0], dst[1]) and np.array_equal(dst[2], dst[1]), (it, args)


def test_table_layout_and_hook(gref, gsim):
    """MpegVideoDSPContext of include/avdsp_b200_tables.h has the reference's layout, and the hook fills exactly the slots
    ff_mpegvideodsp_init fills"""
    from libav_b200 import tables
    out = (C.c_int * 3)()
    gref.ref_mpegvideodsp_layout(out)
    assert list(out) == [C.sizeof(tables.MpegVideoDSPContext), tables.MpegVideoDSPContext.gmc1.offset, tables.MpegVideoDSPContext.gmc.offset]
    ours, theirs = _slot_tables(gsim.ff_mpegvideodsp_init_cuda, gref)
    for name, _ in tables.MpegVideoDSPContext._fields_:
        assert bool(C.cast(getattr(ours, name), C.c_void_p).value) == bool(C.cast(getattr(theirs, name), C.c_void_p).value), name


def test_header_layouts(built, tmp_path):
    """include/avdsp_b200.h as C compiles it: FFMpvMCRecord keeps 44 bytes with mcsel at 42, and FFMpvMCPicture's sprite fields and
    MpegVideoDSPContext sit where libav_b200/tables.py and tests/mpv_gmc_cases.py put them"""
    from libav_b200 import tables
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    src = tmp_path / "probe.c"
    src.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "avdsp_b200.h"\nint main(void) { printf("%d %d %d %d %d %d %d %d %d", '
                   '(int)sizeof(FFMpvMCRecord), (int)offsetof(FFMpvMCRecord, mcsel), (int)sizeof(FFMpvMCPicture), '
                   '(int)offsetof(FFMpvMCPicture, sprite_warping_accuracy), (int)offsetof(FFMpvMCPicture, sprite_offset), '
                   '(int)offsetof(FFMpvMCPicture, sprite_delta), (int)sizeof(MpegVideoDSPContext), (int)offsetof(MpegVideoDSPContext, gmc1), '
                   '(int)offsetof(MpegVideoDSPContext, gmc)); return 0; }\n')
    exe = str(tmp_path / "probe")
    subprocess.check_call(["gcc", "-std=c99", "-Wall", "-Werror", "-I", os.path.join(root, "include"), str(src), "-o", exe])
    mine = [int(x) for x in subprocess.check_output([exe]).split()]
    P, T = tables.FFMpvMCPicture, tables.MpegVideoDSPContext
    assert mine == [G.REC.itemsize, G.REC.fields["mcsel"][1], C.sizeof(P), P.sprite_warping_accuracy.offset, P.sprite_offset.offset,
                    P.sprite_delta.offset, C.sizeof(T), T.gmc1.offset, T.gmc.offset]
