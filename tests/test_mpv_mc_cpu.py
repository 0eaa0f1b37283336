"""CPU: the mpegvideo motion compensation (libav_b200/csrc/mpv_mc.cu + mpv_mc_block.cuh) compiled for the host (tests/hostsim/mpv_mc_hostsim.cpp)
against the reference's own ff_mpv_motion (libavcodec/mpegvideo_motion.c, oracle/_ref/libmpvmcref.so), whole reconstructed frames byte for
byte: every mv_type of both families, field pictures of both parities, first and second fields, forward / backward / bidirectional
records, no_rounding 0 and 1, the quarter-sample chroma workarounds, vectors far outside / at / one step inside every edge, MPEG-4
pictures whose size is not a multiple of 16, H.263 custom sizes whose edges lie past width / height.  Every buffer's padding holds random
bytes.  The plain-C port (oracle/port/orc_mpvmc.c) is pinned to the same reference on the same cases.  Also: the shim runs the real
ff_mpv_motion, records the kernel does not take are counted and leave their macroblock alone, and a picture asking for a refused feature,
or pictures of one call that write the same frame or read each other, change nothing."""
import ctypes as C

import numpy as np
import pytest

import hostsim_build
import mpv_mc_cases as M

# (out_format, structure, first_field, b, no_rnd, qpel, bugs, ragged: 1 MPEG-4 size not a multiple of 16, 2 H.263 custom size)
SCENARIOS = {
    "mpeg2_frame_p": (0, M.FRAME, 1, 0, 0, 0, 0, 0),
    "mpeg2_frame_p_no_rounding": (0, M.FRAME, 1, 0, 1, 0, 0, 0),
    "mpeg2_frame_b": (0, M.FRAME, 1, 1, 0, 0, 0, 0),
    "mpeg2_top_first_p": (0, M.TOP, 1, 0, 0, 0, 0, 0),
    "mpeg2_bottom_first_p": (0, M.BOTTOM, 1, 0, 0, 0, 0, 0),
    "mpeg2_top_second_p": (0, M.TOP, 0, 0, 0, 0, 0, 0),
    "mpeg2_bottom_second_p": (0, M.BOTTOM, 0, 0, 0, 0, 0, 0),
    "mpeg2_top_first_b": (0, M.TOP, 1, 1, 0, 0, 0, 0),
    "mpeg2_bottom_first_b": (0, M.BOTTOM, 1, 1, 0, 0, 0, 0),
    "mpeg2_bottom_second_b": (0, M.BOTTOM, 0, 1, 0, 0, 0, 0),
    "h263_hpel_p": (2, M.FRAME, 1, 0, 0, 0, 0, 0),
    "h263_hpel_p_no_rounding": (2, M.FRAME, 1, 0, 1, 0, 0, 0),
    "mpeg4_hpel_p_ragged": (2, M.FRAME, 1, 0, 1, 0, 0, 1),
    "mpeg4_hpel_b_ragged": (2, M.FRAME, 1, 1, 1, 0, 0, 1),
    "mpeg4_qpel_p_ragged": (2, M.FRAME, 1, 0, 0, 1, 0, 1),
    "mpeg4_qpel_p_no_rounding": (2, M.FRAME, 1, 0, 1, 1, 0, 1),
    "mpeg4_qpel_p_bug_chroma": (2, M.FRAME, 1, 0, 0, 1, M.BUG_QPEL_CHROMA, 1),
    "mpeg4_qpel_p_bug_chroma2": (2, M.FRAME, 1, 0, 1, 1, M.BUG_QPEL_CHROMA2, 0),
    "mpeg4_qpel_p_both_bugs": (2, M.FRAME, 1, 0, 0, 1, M.BUG_QPEL_CHROMA | M.BUG_QPEL_CHROMA2, 1),
    "mpeg4_qpel_b_ragged": (2, M.FRAME, 1, 1, 0, 1, 0, 1),
    "h263_custom_size_hpel_p": (2, M.FRAME, 1, 0, 1, 0, 0, 2),
    "h263_custom_size_qpel_p": (2, M.FRAME, 1, 0, 0, 1, 0, 2),
    "h263_custom_size_qpel_b": (2, M.FRAME, 1, 1, 0, 1, M.BUG_QPEL_CHROMA, 2),
}


def scenario_picture(name, seed, mb_w=7, mb_h=6, refs=None):
    fmt, st, ff, b, nr, qp, bugs, ragged = SCENARIOS[name]
    rng = np.random.default_rng(seed)
    kw = dict(width=16 * mb_w - 5, height=16 * mb_h - 3, custom_edges=ragged == 2) if ragged else {}
    pic = M.Picture(rng, fmt, mb_w, mb_h, structure=st, first_field=ff, b=b, no_rnd=nr, qpel=qp, bugs=bugs, refs=refs, **kw)
    M.make_records(rng, pic)
    return pic


@pytest.fixture(scope="session")
def mcref(built):
    lib = M.ref_lib()
    if lib is None:
        pytest.skip("oracle/_ref not built (no reference tree in this environment)")
    return lib


@pytest.fixture
def mcsim(built):
    return hostsim_build.fresh()


@pytest.fixture(scope="session")
def mcport(built):
    return M.port_lib()


def test_shim_runs_the_real_ff_mpv_motion(mcref):
    """libavref.so exports an aborting stand-in named ff_mpv_motion; the shim's function is another one, and a zero vector copies the
    reference macroblock (the stand-in would have ended the process)"""
    real, stub = C.c_void_p(), C.c_void_p()
    mcref.ref_mpvmc_impl(C.byref(real), C.byref(stub))
    assert real.value and stub.value and real.value != stub.value
    pic = M.Picture(np.random.default_rng(1), 0, 3, 2)
    pic.recs = np.zeros(1, M.REC)
    pic.recs[0]["mb_x"], pic.recs[0]["mb_y"], pic.recs[0]["mv_dir"] = 1, 1, 1
    out = M.run_ref(mcref, pic)
    assert np.array_equal(out[0][16:32, 16:32], pic.last[0][16:32, 16:32])
    assert np.array_equal(out[1][8:16, 8:16], pic.last[1][8:16, 8:16])
    assert np.array_equal(out[0][:16], pic.frame[0][:16])


@pytest.mark.parametrize("seed", [1, 2, 3])
@pytest.mark.parametrize("name", list(SCENARIOS))
def test_hostsim_matches_reference(mcref, mcsim, name, seed):
    pic = scenario_picture(name, 100 * seed + len(name))
    want = M.run_ref(mcref, pic)
    got, rej = M.run_sim(mcsim, [pic])
    assert rej == 0
    d = M.first_diff(got[0], want)
    assert d is None, (name, d)


@pytest.mark.parametrize("fmt,structure,custom", [(0, M.FRAME, 0), (0, M.TOP, 0), (2, M.FRAME, 0), (2, M.FRAME, 1)])
def test_every_type_and_edge_exhaustively(mcref, mcsim, fmt, structure, custom):
    """a small picture where every macroblock touches an edge, each type alone, every record near an edge or far outside; in the
    H.263 family also with the custom-size edges (h_edge_pos above width), where the clip of a 4MV block to width reads directly"""
    for t in M.mv_types(fmt, structure):
        for qpel in ((0, 1) if fmt == 2 else (0,)):
            for seed in range(4):
                rng = np.random.default_rng(seed * 10 + t)
                pic = M.Picture(rng, fmt, 3, 2, structure=structure, first_field=seed & 1, b=seed >> 1, no_rnd=seed & 1, qpel=qpel,
                                width=43 if fmt == 2 else None, height=29 if fmt == 2 else None, custom_edges=bool(custom))
                M.make_records(rng, pic, far=0.3, edge=0.6, types=[t])
                want = M.run_ref(mcref, pic)
                got, rej = M.run_sim(mcsim, [pic])
                assert rej == 0 and M.first_diff(got[0], want) is None, (t, qpel, seed, M.first_diff(got[0], want))


@pytest.mark.parametrize("qpel", [0, 1])
def test_tiny_pictures_read_one_past_the_aligned_plane(mcref, mcsim, qpel):
    """h_edge_pos below 16: FFMAX(h_edge_pos - 16, 0) = 0 lets a 16x16 vector read the reference directly, and its chroma block then
    reads column 8 of a one-macroblock-wide picture, one past the macroblock-aligned plane (the row below likewise)"""
    for seed in range(40):
        rng = np.random.default_rng(seed)
        w, h = int(rng.integers(2, 16)), int(rng.integers(2, 16))
        pic = M.Picture(rng, 2, 1, 1, no_rnd=seed & 1, qpel=qpel, bugs=[0, M.BUG_QPEL_CHROMA, M.BUG_QPEL_CHROMA2][seed % 3], width=w, height=h)
        pic.recs = np.zeros(1, M.REC)
        pic.recs[0]["mv_dir"] = 1
        pic.recs[0]["mv"][0, 0] = rng.integers(0, 4, 2)
        want = M.run_ref(mcref, pic)
        got, rej = M.run_sim(mcsim, [pic])
        assert rej == 0 and M.first_diff(got[0], want) is None, (seed, w, h, M.first_diff(got[0], want))


def test_stacked_pictures_in_one_call(mcref, mcsim):
    """pictures of both families in one call, sharing reference frames; each equals the reference run on its own"""
    pics = []
    shared = None
    for i, name in enumerate(["mpeg2_frame_b", "mpeg2_top_first_p", "mpeg4_qpel_b_ragged", "mpeg2_frame_p"]):
        pic = scenario_picture(name, 40 + i, refs=shared if name.startswith("mpeg2_frame") else None)
        if name == "mpeg2_frame_b":
            shared = (pic.last, pic.next)
        pics.append(pic)
    got, rej = M.run_sim(mcsim, pics)
    assert rej == 0
    for pic, g in zip(pics, got):
        assert M.first_diff(g, M.run_ref(mcref, pic)) is None


def bad_records(pic, rng):
    """records the kernel does not take: outside the picture, mv_type out of range or not in the family, mv_dir above 7"""
    recs = pic.recs.copy()
    n = len(recs)
    idx = rng.permutation(n)[: n // 3]
    for j, i in enumerate(idx):
        kind = j % 4
        if kind == 0:
            recs[i]["mb_x"] = pic.p["mb_width"] + int(rng.integers(0, 60000 - pic.p["mb_width"]))
        elif kind == 1:
            recs[i]["mb_y"] = pic.mb_rows + int(rng.integers(0, 3))
        elif kind == 2:
            recs[i]["mv_type"] = int(rng.choice([5, 9, 255] + ([M.TFIELD, M.T16X8, M.TDMV] if pic.p["out_format"] == 2 else [M.T8X8])))
        else:
            recs[i]["mv_dir"] = int(rng.choice([8, 9, 255]))
    return recs


@pytest.mark.parametrize("name", ["mpeg2_frame_b", "mpeg2_bottom_second_p", "mpeg4_qpel_b_ragged"])
def test_rejected_records_are_counted_and_untouched(mcref, mcsim, name):
    rng = np.random.default_rng(5)
    pic = scenario_picture(name, 77)
    pic.recs = bad_records(pic, rng)
    n_bad = int((~pic.accepted()).sum())
    assert n_bad > 0
    want = M.run_ref(mcref, pic)                 # the reference runs the accepted records only
    got, rej = M.run_sim(mcsim, [pic])
    assert rej == n_bad
    assert M.first_diff(got[0], want) is None


REFUSALS = [("obmc", 1), ("sprite", 1), ("mspel", 1), ("lowres", 1), ("chroma_format", 2), ("out_format", 1), ("out_format", 3),
            ("picture_structure", 0), ("h_edge_pos", 0), ("mb_width", 0), ("pic_linesize", 7)]


@pytest.mark.parametrize("field,value", REFUSALS)
def test_picture_level_refusal(mcsim, field, value):
    pic = scenario_picture("mpeg4_qpel_p_ragged", 3)
    frame = [a.copy() for a in pic.frame]
    recs = np.ascontiguousarray(pic.recs)
    base = [a.ctypes.data for a in frame]
    s = M.picture_struct(pic, base, base, [a.ctypes.data for a in pic.last], [a.ctypes.data for a in pic.next], recs.ctypes.data, len(recs))
    setattr(s, field, value)
    rej = np.zeros(1, np.uint32)
    mcsim.avb200_clear_error()
    assert mcsim.ff_mpv_motion_batch_cuda(C.byref(s), 1, rej.ctypes.data, None) == -1
    assert mcsim.avb200_last_error()
    assert all(np.array_equal(a, b) for a, b in zip(frame, pic.frame)) and rej[0] == 0


def test_h263_field_picture_and_pictures_reading_each_other_are_refused(mcsim):
    pic = scenario_picture("mpeg2_top_first_p", 3)
    other = scenario_picture("mpeg2_bottom_second_p", 4)
    frame = [a.ctypes.data for a in pic.frame]
    a = M.picture_struct(pic, frame, frame, [x.ctypes.data for x in pic.last], [x.ctypes.data for x in pic.next], pic.recs.ctypes.data, len(pic.recs))
    # the second field of the same frame in the same call
    b = M.picture_struct(other, frame, frame, [x.ctypes.data for x in pic.last], [x.ctypes.data for x in pic.next], other.recs.ctypes.data, len(other.recs))
    arr = (type(a) * 2)(a, b)
    rej = np.zeros(1, np.uint32)
    mcsim.avb200_clear_error()
    assert mcsim.ff_mpv_motion_batch_cuda(C.cast(arr, C.c_void_p), 2, rej.ctypes.data, None) == -1
    assert b"read each other" in mcsim.avb200_last_error()
    a.out_format = 2
    mcsim.avb200_clear_error()
    assert mcsim.ff_mpv_motion_batch_cuda(C.byref(a), 1, rej.ctypes.data, None) == -1
    assert b"field pictures" in mcsim.avb200_last_error()


# ------------------------------------------------------------------------------------------------------------------------ the port

@pytest.mark.parametrize("seed", [1, 2])
@pytest.mark.parametrize("name", list(SCENARIOS))
def test_port_matches_reference(mcref, mcport, name, seed):
    """oracle/port/orc_mpvmc.c (block operations, emulated edges copied into a buffer) against the unmodified mpegvideo_motion.c"""
    pic = scenario_picture(name, 300 * seed + len(name))
    d = M.first_diff(M.run_ref(mcport, pic), M.run_ref(mcref, pic))
    assert d is None, (name, d)


@pytest.mark.parametrize("fmt,structure,custom", [(0, M.FRAME, 0), (0, M.BOTTOM, 0), (2, M.FRAME, 0), (2, M.FRAME, 1)])
def test_port_every_type_near_edges(mcref, mcport, fmt, structure, custom):
    for t in M.mv_types(fmt, structure):
        for qpel in ((0, 1) if fmt == 2 else (0,)):
            for seed in range(6):
                rng = np.random.default_rng(seed * 10 + t + 7)
                pic = M.Picture(rng, fmt, 3, 2, structure=structure, first_field=seed & 1, b=(seed >> 1) & 1, no_rnd=seed & 1, qpel=qpel,
                                width=43 if fmt == 2 else None, height=29 if fmt == 2 else None, custom_edges=bool(custom))
                M.make_records(rng, pic, far=0.3, edge=0.6, types=[t])
                assert M.first_diff(M.run_ref(mcport, pic), M.run_ref(mcref, pic)) is None, (t, qpel, seed)


@pytest.mark.parametrize("qpel", [0, 1])
def test_port_tiny_pictures(mcref, mcport, qpel):
    for seed in range(40):
        rng = np.random.default_rng(seed)
        pic = M.Picture(rng, 2, 1, 1, no_rnd=seed & 1, qpel=qpel, bugs=[0, M.BUG_QPEL_CHROMA, M.BUG_QPEL_CHROMA2][seed % 3],
                        width=int(rng.integers(2, 16)), height=int(rng.integers(2, 16)))
        pic.recs = np.zeros(1, M.REC)
        pic.recs[0]["mv_dir"] = 1
        pic.recs[0]["mv"][0, 0] = rng.integers(0, 4, 2)
        assert M.first_diff(M.run_ref(mcport, pic), M.run_ref(mcref, pic)) is None, seed


def test_conflicts_are_found_by_frame_base_without_cur(mcsim):
    """cur is optional for frame pictures: a picture whose destination frame is another's reference, or its own reference, is still
    refused, and nothing is run"""
    a, b = scenario_picture("mpeg2_frame_p", 5), scenario_picture("mpeg2_frame_b", 6)
    fa = [x.copy() for x in a.frame]
    base_a = [x.ctypes.data for x in fa]
    sa = M.picture_struct(a, base_a, [0, 0, 0], [x.ctypes.data for x in a.last], [x.ctypes.data for x in a.next], a.recs.ctypes.data, len(a.recs))
    # b predicts from a's frame
    sb = M.picture_struct(b, [x.ctypes.data for x in b.frame], [0, 0, 0], base_a, [x.ctypes.data for x in b.next], b.recs.ctypes.data, len(b.recs))
    for s in (sa, sb):
        for i in range(3):
            s.cur[i] = None
    rej = np.zeros(1, np.uint32)
    arr = (type(sa) * 2)(sa, sb)
    mcsim.avb200_clear_error()
    assert mcsim.ff_mpv_motion_batch_cuda(C.cast(arr, C.c_void_p), 2, rej.ctypes.data, None) == -1
    assert b"read each other" in mcsim.avb200_last_error()
    own = M.picture_struct(a, base_a, [0, 0, 0], base_a, [x.ctypes.data for x in a.next], a.recs.ctypes.data, len(a.recs))
    for i in range(3):
        own.cur[i] = None
    mcsim.avb200_clear_error()
    assert mcsim.ff_mpv_motion_batch_cuda(C.byref(own), 1, rej.ctypes.data, None) == -1
    assert b"being reconstructed" in mcsim.avb200_last_error()
    assert all(np.array_equal(x, y) for x, y in zip(fa, a.frame)) and rej[0] == 0
