"""CPU: the H.263 deblocking filter.  The product's picture filter (libav_b200/csrc/h263_lf.cuh) compiled for the host
(tests/hostsim/h263_hostsim.cpp) and its two-pass plain-C restatement (oracle/port/orc_h263.c) against the reference's serial driver --
ff_h263_loop_filter for every macroblock in raster order, libavcodec/h263.c with h263dsp.c, oracle/_ref/libh263ref.so -- whole buffers
byte for byte, padding included: random pictures with random skip flags and qscale 1..31, mostly and wholly skipped pictures, both
chroma qscale tables, 1 x N, N x 1 and 1 x 1 macroblock pictures, several pictures per call.  The port matching the serial driver is the
proof that every horizontal edge, then every vertical edge, with each edge's qp taken from its two macroblocks, gives the serial result.
Also: the H263DSPContext slots (their kernel on the host, and the port) against the reference's C functions over qscale 0..31, every
range of the filter's d, both stride signs, with the bytes around the call compared too; the table layout and what the hook fills; and
the refusals, which return -1 and change nothing."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

import h263_cases as H

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def lfref(built):
    lib = H.ref_lib()
    if lib is None:
        pytest.skip("oracle/_ref not built (no reference tree in this environment)")
    return lib


@pytest.fixture(scope="module")
def lfsim(built):
    return H.sim_lib()


@pytest.fixture(scope="module")
def lfport(built):
    return H.port_lib()


SHAPES = [(7, 6), (11, 9), (22, 18), (1, 5), (5, 1), (1, 1), (2, 2), (3, 1), (1, 3)]


def cases(seed):
    rng = np.random.default_rng(seed)
    for k, (w, h) in enumerate(SHAPES):
        for skip in (0.0, 0.3, 0.9, 1.0):
            chroma = H.ANNEX_T_CHROMA_QSCALE if (k + int(10 * skip)) % 2 else None
            yield "%dx%d skip %.1f %s" % (w, h, skip, "annex T" if chroma is not None else "default"), H.LfPicture(rng, w, h, skip=skip, chroma=chroma)


@pytest.mark.parametrize("seed", [1, 2, 3])
def test_port_two_passes_match_the_serial_reference(lfref, lfport, seed):
    for name, pic in cases(seed):
        d = H.first_diff(H.run_serial(lfport, pic), H.run_serial(lfref, pic))
        assert d is None, (name, d)


@pytest.mark.parametrize("seed", [1, 2, 3])
def test_hostsim_matches_the_serial_reference(lfref, lfsim, seed):
    for name, pic in cases(seed):
        d = H.first_diff(H.run_sim(lfsim, [pic])[0], H.run_serial(lfref, pic))
        assert d is None, (name, d)


def test_filter_changes_the_picture(lfref):
    """the comparisons above are not vacuous: a picture with no skipped macroblock changes, an all-skipped one does not"""
    rng = np.random.default_rng(4)
    pic = H.LfPicture(rng, 6, 5, skip=0.0)
    out = H.run_serial(lfref, pic)
    assert all(not np.array_equal(o, b) for o, b in zip(out, pic.bufs))
    pic = H.LfPicture(rng, 6, 5, skip=1.0)
    assert all(np.array_equal(o, b) for o, b in zip(H.run_serial(lfref, pic), pic.bufs))


def test_hostsim_custom_sizes_and_odd_strides(lfref, lfsim):
    """linesizes that are not multiples of 4 (the kernel's byte path), a larger mb_stride, low and high qscale ranges"""
    rng = np.random.default_rng(9)
    for i in range(12):
        w, h = int(rng.integers(1, 12)), int(rng.integers(1, 10))
        pic = H.LfPicture(rng, w, h, skip=float(rng.random()), extra_cols=int(rng.integers(0, 9)), mb_stride=w + 1 + int(rng.integers(0, 4)),
                          qmin=[1, 1, 20][i % 3], qmax=[31, 4, 31][i % 3], chroma=H.ANNEX_T_CHROMA_QSCALE if i & 1 else None)
        d = H.first_diff(H.run_sim(lfsim, [pic])[0], H.run_serial(lfref, pic))
        assert d is None, (i, w, h, d)


def test_hostsim_stacked_pictures_in_one_call(lfref, lfsim):
    """more pictures than one launch carries (16), of different sizes; each equals the reference run on its own"""
    rng = np.random.default_rng(11)
    pics = [H.LfPicture(rng, int(rng.integers(1, 9)), int(rng.integers(1, 7)), skip=float(rng.random()),
                        chroma=H.ANNEX_T_CHROMA_QSCALE if i % 3 == 0 else None) for i in range(19)]
    for i, (g, pic) in enumerate(zip(H.run_sim(lfsim, pics), pics)):
        assert H.first_diff(g, H.run_serial(lfref, pic)) is None, i


# ---------------------------------------------------------------------------------------------------------------------------- refusals

def refusal_cases(rng):
    """(name, pictures, mutate(array)) triples"""
    def bad(field, value):
        def f(arr):
            setattr(arr[0], field, value)
        return f

    def null_plane(arr):
        arr[0].data[2] = None

    def null_table(arr):
        arr[0].qscale_table = None

    def chroma_entry(arr):
        arr[0].chroma_qscale_table[5] = 32

    yield "mb_width 0", bad("mb_width", 0)
    yield "mb_height 0", bad("mb_height", 0)
    yield "mb_width above 4096", bad("mb_width", 4097)
    yield "mb_stride = mb_width", bad("mb_stride", 6)
    yield "linesize below the aligned width", bad("linesize", 95)
    yield "uvlinesize below the aligned width", bad("uvlinesize", 47)
    yield "negative linesize", bad("linesize", -96)
    yield "NULL plane", null_plane
    yield "NULL qscale_table", null_table
    yield "chroma qscale above 31", chroma_entry


def test_refusals_change_nothing(lfsim):
    rng = np.random.default_rng(3)
    for name, mutate in refusal_cases(rng):
        pics = [H.LfPicture(rng, 6, 4, skip=0.0, extra_cols=0), H.LfPicture(rng, 3, 3, skip=0.0)]
        bufs = [[a.copy() for a in p.bufs] for p in pics]
        arr = H.host_structs(pics, bufs)
        mutate(arr)
        lfsim.hostsim_clear_error()
        assert lfsim.ff_h263_loop_filter_batch_cuda(C.cast(arr, C.c_void_p), 2, None) == -1, name
        assert lfsim.hostsim_last_error(), name
        assert all(np.array_equal(a, b) for bb, p in zip(bufs, pics) for a, b in zip(bb, p.bufs)), name


def test_pictures_sharing_a_frame_are_refused(lfsim):
    rng = np.random.default_rng(5)
    pics = [H.LfPicture(rng, 4, 3, skip=0.0), H.LfPicture(rng, 4, 3, skip=0.0), H.LfPicture(rng, 2, 2, skip=0.0)]
    bufs = [[a.copy() for a in p.bufs] for p in pics]
    for share in ("same frame", "chroma inside another's luma"):
        arr = H.host_structs(pics, bufs)
        if share == "same frame":
            arr[2] = arr[0]
        else:
            arr[2].data[1] = arr[1].data[0] + 5 * pics[1].ls
        lfsim.hostsim_clear_error()
        assert lfsim.ff_h263_loop_filter_batch_cuda(C.cast(arr, C.c_void_p), 3, None) == -1
        assert b"share a frame" in lfsim.hostsim_last_error()
        assert all(np.array_equal(a, b) for bb, p in zip(bufs, pics) for a, b in zip(bb, p.bufs))
    lfsim.hostsim_clear_error()
    assert lfsim.ff_h263_loop_filter_batch_cuda(None, 0, None) == 0
    assert lfsim.ff_h263_loop_filter_batch_cuda(None, 2, None) == -1


def test_flush_refuses_a_bad_loop_filter_picture_before_anything_runs(lfsim):
    """the flush checks its loop-filter pictures before the first stage: a bad one leaves even the motion compensation undone"""
    import mpv_mc_cases as M
    from libav_b200 import tables
    rng = np.random.default_rng(8)
    pic = M.Picture(rng, 2, 4, 3)
    M.make_records(rng, pic)
    frame = [a.copy() for a in pic.frame]
    base = [a.ctypes.data for a in frame]
    recs = np.ascontiguousarray(pic.recs)
    mc = M.picture_struct(pic, base, base, [a.ctypes.data for a in pic.last], [a.ctypes.data for a in pic.next], recs.ctypes.data, len(recs))
    lp = H.LfPicture(rng, 4, 3)
    lbufs = [a.copy() for a in lp.bufs]
    larr = H.host_structs([lp], [lbufs])
    larr[0].mb_stride = 2
    rej = np.zeros(1, np.uint32)
    w = tables.FFMpvPictureWork()
    w.pictures, w.n_pictures, w.rejected = C.cast(C.pointer(mc), C.c_void_p), 1, rej.ctypes.data
    w.loop_filter, w.n_loop_filter = C.cast(larr, C.c_void_p), 1
    lfsim.hostsim_clear_error()
    assert lfsim.ff_mpv_flush_pictures_cuda(C.byref(w), None) == -1
    assert b"mb_stride" in lfsim.hostsim_last_error()
    assert all(np.array_equal(a, b) for a, b in zip(frame, pic.frame)) and all(np.array_equal(a, b) for a, b in zip(lbufs, lp.bufs))


def test_flush_runs_motion_compensation_then_the_loop_filter(lfref, lfsim):
    """a flush without residual batches on an H.263 custom-size picture: the reference motion compensation, then the serial reference
    loop filter over its result"""
    import mpv_mc_cases as M
    from libav_b200 import tables
    rng = np.random.default_rng(12)
    pic = M.Picture(rng, 2, 5, 4, no_rnd=1, width=75, height=61, custom_edges=True)
    M.make_records(rng, pic)
    tabs = H.LfPicture(rng, 5, 4, skip=0.3, chroma=H.ANNEX_T_CHROMA_QSCALE)       # its mb_type / qscale_table / chroma table only
    ls, uvls = pic.p["linesize"], pic.p["uvlinesize"]
    frame = [a.copy() for a in pic.frame]
    recs = np.ascontiguousarray(pic.recs)
    base = [a.ctypes.data for a in frame]
    mc = M.picture_struct(pic, base, base, [a.ctypes.data for a in pic.last], [a.ctypes.data for a in pic.next], recs.ctypes.data, len(recs))
    lf = tables.FFH263LoopFilterPicture()
    for k in range(3):
        lf.data[k] = base[k]
    lf.linesize, lf.uvlinesize, lf.mb_width, lf.mb_height, lf.mb_stride = ls, uvls, 5, 4, tabs.mb_stride
    lf.mb_type, lf.qscale_table = tabs.mb_type.ctypes.data, tabs.qscale.ctypes.data
    lf.chroma_qscale_table[:] = [int(x) for x in tabs.chroma]
    rej = np.zeros(1, np.uint32)
    w = tables.FFMpvPictureWork()
    w.pictures, w.n_pictures, w.rejected = C.cast(C.pointer(mc), C.c_void_p), 1, rej.ctypes.data
    w.loop_filter, w.n_loop_filter = C.cast(C.pointer(lf), C.c_void_p), 1
    assert lfsim.ff_mpv_flush_pictures_cuda(C.byref(w), None) == 0, lfsim.hostsim_last_error()
    mcd = M.run_ref(M.ref_lib(), pic)
    want = [a.copy() for a in mcd]
    prm = np.array([ls, uvls, 5, 4, tabs.mb_stride], np.int32)
    ct = np.ascontiguousarray(tabs.chroma, np.uint8)
    assert lfref.picture((C.c_void_p * 3)(*[a.ctypes.data for a in want]), prm.ctypes.data, tabs.mb_type.ctypes.data, tabs.qscale.ctypes.data,
                         ct.ctypes.data) == 0
    assert not all(np.array_equal(x, y) for x, y in zip(want, mcd))
    assert M.first_diff(frame, want) is None and rej[0] == 0


# ---------------------------------------------------------------------------------------------------------------------------- the slots

class _RefSlots:
    def __init__(self, lib):
        from libav_b200 import tables
        self.t = tables.H263DSPContext()
        lib.ref_h263dsp_init(C.byref(self.t))
        self.h, self.v = self.t.h263_h_loop_filter, self.t.h263_v_loop_filter


def slot_sweep(callee, want_callee):
    """every qscale, every d range, both strides, both directions; the whole 12 x 12 buffer compared"""
    rng = np.random.default_rng(21)
    n = 0
    for vert in (0, 1):
        for sign in (1, -1):
            for q in range(32):
                for dk in range(4):
                    buf, off, stride = H.slot_case(rng, vert, sign, q, dk)
                    a, b = buf.copy(), buf.copy()
                    callee(vert, a, off, stride, q)
                    want_callee(vert, b, off, stride, q)
                    assert np.array_equal(a, b), (vert, sign, q, dk)
                    n += not np.array_equal(b, buf)
    assert n > 300           # most calls change samples


def test_slot_kernel_matches_reference(lfref, lfsim):
    r = _RefSlots(lfref)
    slot_sweep(lambda v, a, o, s, q: lfsim.hostsim_h263_slot(v, a.ctypes.data + o, s, q),
               lambda v, b, o, s, q: (r.h if v else r.v)(C.cast(b.ctypes.data + o, C.POINTER(C.c_uint8)), s, q))


def test_port_slots_match_reference(lfref, lfport):
    r = _RefSlots(lfref)
    slot_sweep(lambda v, a, o, s, q: (lfport.h_loop_filter if v else lfport.v_loop_filter)(a.ctypes.data + o, s, q),
               lambda v, b, o, s, q: (r.h if v else r.v)(C.cast(b.ctypes.data + o, C.POINTER(C.c_uint8)), s, q))


def test_h263dsp_layout_and_hook(lfref, built, tmp_path):
    """H263DSPContext of include/avdsp_b200_tables.h has the reference's layout, and the hook fills exactly the slots ff_h263dsp_init
    fills (without a GPU the slots are only installed, not called)"""
    import libav_b200._lib as L
    from libav_b200 import tables
    info = (C.c_int * 3)()
    lfref.ref_h263_abi_info(info)
    src = tmp_path / "probe.c"
    src.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "avdsp_b200.h"\nint main(void) { printf("%d %d %d", (int)sizeof(H263DSPContext), '
                   '(int)offsetof(H263DSPContext, h263_h_loop_filter), (int)offsetof(H263DSPContext, h263_v_loop_filter)); return 0; }\n')
    exe = str(tmp_path / "probe")
    subprocess.check_call(["gcc", "-std=c99", "-Wall", "-Werror", "-I", os.path.join(ROOT, "include"), str(src), "-o", exe])
    mine = [int(x) for x in subprocess.check_output([exe]).split()]
    assert mine == list(info)
    assert [C.sizeof(tables.H263DSPContext), tables.H263DSPContext.h263_h_loop_filter.offset, tables.H263DSPContext.h263_v_loop_filter.offset] == mine
    ref_t, ours = tables.H263DSPContext(), tables.H263DSPContext()
    lfref.ref_h263dsp_init(C.byref(ref_t))
    L.lib.ff_h263dsp_init_cuda(C.byref(ours))
    for name, _ in tables.H263DSPContext._fields_:
        assert bool(C.cast(getattr(ref_t, name), C.c_void_p).value) == bool(C.cast(getattr(ours, name), C.c_void_p).value), name
