"""ProRes reconstruction (libav_b200/csrc/prores.cu) compiled as host C++ (tests/hostsim/prores_hostsim.cpp) against the reference
(oracle/_ref/libproresref.so: proresdsp.c, simple_idct.c, proresdec.c, proresenc.c, unmodified): the ProresDSPContext slot and the batch call
on edge blocks, and the picture call on reference-encoded streams.  Also the table's layout against the reference's, the hook's fill against
ff_proresdsp_init's, and the public header against the library's exports and the ctypes mirrors."""
import ctypes as C
import os
import re
import subprocess

import numpy as np
import pytest

import hostsim_build
import prores_util as U
from libav_b200 import tables

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)


@pytest.fixture(scope="session")
def pref(built):
    lib = U.ref()
    if lib is None:
        pytest.skip("oracle/_ref not built (no reference tree in this environment)")
    return lib


@pytest.fixture(scope="session")
def hs(built):
    return hostsim_build.load()


def test_edge_blocks_slot(hs, pref):
    """ff_proresdsp_init_cuda's idct_put against prores_idct_put_c: the samples and the block it leaves, at odd and even line sizes"""
    t = tables.ProresDSPContext()
    hs.ff_proresdsp_init_cuda(C.byref(t))
    blocks, qm, qidx = U.edge_blocks(1)
    want_b, want_s = U.ref_idct_put(pref, blocks, qm, qidx)
    for k in range(0, len(blocks), 3):
        b = blocks[k].copy()
        for ls in (16, 40, 41):
            out = np.full(8 * ls // 2 + 8, 0x7777, np.uint16)
            bb = b.copy()
            t.idct_put(out.ctypes.data_as(C.POINTER(C.c_uint16)), ls, bb.ctypes.data_as(C.POINTER(C.c_int16)),
                       qm[k].ctypes.data_as(C.POINTER(C.c_int16)))
            ref_out = np.full_like(out, 0x7777)
            rb = b.copy()
            pref.ref_prores_idct_put(U.P(ref_out), ls, U.P(rb), U.P(qm[k]))
            assert np.array_equal(out, ref_out) and np.array_equal(bb, rb), (k, ls)
        assert np.array_equal(rb, want_b[k])
    assert hs.avb200_last_error() in (b"", None)


@pytest.mark.parametrize("layout", ["aligned", "odd_pitch", "unaligned_blocks", "no_qidx"])
def test_edge_blocks_batch(hs, pref, layout):
    """the batch call (its thread-per-block kernel here): samples and final blocks equal prores_idct_put_c's on every edge block"""
    blocks, qm, qidx = U.edge_blocks(2)
    if layout == "no_qidx":
        qidx, qm = np.zeros(len(blocks), np.uint32), qm[7:8]
    want_b, want_s = U.ref_idct_put(pref, blocks, qm, qidx)
    kw = {"odd_pitch": dict(pitch_extra=2), "unaligned_blocks": dict(block_pad=2, qmat_pad=2)}.get(layout, {})
    rc, got_b, got_s = U.run_batch(hs, U.HostMem(), blocks, qm, None if layout == "no_qidx" else qidx, **kw)
    assert rc == 0
    assert np.array_equal(got_b, want_b), np.flatnonzero((got_b != want_b).any(1))[:8]
    assert np.array_equal(got_s, want_s), np.flatnonzero((got_s != want_s).reshape(len(blocks), -1).any(1))[:8]


def test_edge_block_coverage(pref):
    """the edge set reaches what it is meant to: both clip bounds, wrapped products, and rows that only dequantisation makes DC-only"""
    blocks, qm, qidx = U.edge_blocks(1)
    _, s = U.ref_idct_put(pref, blocks, qm, qidx)
    assert (s == 4).any() and (s == 1019).any()
    prod = blocks.astype(np.int64) * qm.astype(np.int64)
    assert ((prod != prod.astype(np.int16)) & (prod.astype(np.int16) == 0)).any()
    assert ((prod < -32768) | (prod > 32767)).any()


@pytest.mark.parametrize("spec", U.SMALL_STREAMS, ids=str)
def test_pictures_match_reference_decoder(hs, pref, spec):
    """the picture call on one reference-encoded frame, every picture of it: y / u / v byte for byte, alpha and padding untouched"""
    d = U.Decoded(pref, spec)
    rc, got = U.run_pictures(hs, U.HostMem(), [d])
    assert rc == 0, hs.avb200_last_error()
    U.check_frame(d, got[0])


def test_pictures_scrambled_quantisers(hs, pref):
    """header matrices of any byte value and slice scale factors up to 512: (int16)(qmat * sf) wraps, as in decode_slice"""
    decs = [U.Decoded(pref, spec, seed=11 + k, scrambled=True) for k, spec in enumerate(U.SMALL_STREAMS[:6])]
    assert any(int(np.max(d.rec.np_ssf)) == 512 for d in decs)
    rc, got = U.run_pictures(hs, U.HostMem(), decs)
    assert rc == 0
    for d, g in zip(decs, got):
        U.check_frame(d, g)


def test_pictures_mixed_geometry_one_call(hs, pref):
    """several pictures of different sizes, chroma formats and field orders in one call"""
    decs = [U.Decoded(pref, spec, seed=20 + k) for k, spec in enumerate(U.SMALL_STREAMS)]
    rc, got = U.run_pictures(hs, U.HostMem(), decs)
    assert rc == 0
    for d, g in zip(decs, got):
        U.check_frame(d, g)


def refusals(base_work):
    """(name, mutate) pairs, each making a valid FFProresPictureWork invalid"""
    def m(**kw):
        def f(w):
            for k, v in kw.items():
                if isinstance(v, tuple):
                    getattr(w, k)[v[0]] = v[1]
                else:
                    setattr(w, k, v)
        return f
    return [
        ("chroma_format_1", m(chroma_format=1)), ("chroma_format_0", m(chroma_format=0)),
        ("slice_width_factor_4", m(slice_width_factor=4)), ("slice_width_factor_neg", m(slice_width_factor=-1)),
        ("null_y", m(data=(0, None))), ("null_v", m(data=(2, None))), ("odd_u", m(data=(1, base_work.data[1] + 1))),
        ("odd_linesize", m(linesize=(0, base_work.linesize[0] + 1))), ("zero_linesize", m(linesize=(2, 0))),
        ("narrow_luma", m(linesize=(0, 32 * base_work.mb_width - 2))), ("narrow_chroma", m(linesize=(1, 8 * base_work.mb_width))),
        ("short_plane", m(mb_rows=(0, base_work.mb_height - 1))), ("short_chroma", m(mb_rows=(2, base_work.mb_height - 1))),
        ("too_few_slices", m(n_slices=base_work.n_slices - 1)), ("too_many_slices", m(n_slices=base_work.n_slices + 1)),
        ("null_slices", m(slices=None)), ("null_blocks", m(blocks=None)), ("mb_width_0", m(mb_width=0)), ("mb_height_0", m(mb_height=0)),
    ]


def check_refusals(lib, mem, d):
    bl = mem.put(U.picture_blocks(d.rec, 0)); sl = mem.put(U.slice_table(d.rec, 0))
    fb = mem.put(d.frame.buf)
    base = U.picture_works(d.frame, d.rec, fb, lambda k: bl, lambda k: sl)[0]
    names = []
    for name, mutate in refusals(base):
        w = tables.FFProresPictureWork.from_buffer_copy(base)
        mutate(w)
        good = tables.FFProresPictureWork.from_buffer_copy(base)
        arr = (tables.FFProresPictureWork * 2)(good, w)                 # the valid picture in front is not written either
        lib.avb200_clear_error()
        assert lib.ff_prores_decode_pictures_cuda(arr, 2, None) == -1, name
        assert b"ff_prores_decode_pictures_cuda" in (lib.avb200_last_error() or b""), name
        names.append(name)
    lib.avb200_clear_error()
    assert lib.ff_prores_decode_pictures_cuda(None, 1, None) == -1 and lib.ff_prores_decode_pictures_cuda(None, -1, None) == -1
    lib.avb200_clear_error()
    assert lib.ff_prores_idct_put_batch_cuda(None, None, None, 16, None, None, 1, None) == -1
    lib.avb200_clear_error()
    assert lib.ff_prores_idct_put_batch_cuda(C.c_void_p(bl), C.c_void_p(fb), C.c_void_p(sl), 17, C.c_void_p(bl), None, 1, None) == -1
    lib.avb200_clear_error()
    mem.sync()
    assert np.array_equal(mem.get(fb, np.uint8, d.frame.buf.shape), d.frame.buf), "a refused call wrote"
    return names


def test_refusals(hs, pref):
    d = U.Decoded(pref, U.SMALL_STREAMS[0])
    assert len(check_refusals(hs, U.HostMem(), d)) == 19


# ------------------------------------------------------------------------------------------------------------------ table and interface

def test_table_layout_matches_reference(pref):
    out = (C.c_long * 4)()
    pref.ref_prores_abi(out)
    T = tables.ProresDSPContext
    assert list(out) == [C.sizeof(T), T.idct_permutation_type.offset, T.idct_permutation.offset, T.idct_put.offset]
    exe = os.path.join(hostsim_build.GEN, "prores_abi_probe.%d" % os.getpid())
    os.makedirs(hostsim_build.GEN, exist_ok=True)
    code = ('#include <stdio.h>\n#include <stddef.h>\n#include "avdsp_b200.h"\nint main(void){printf("%ld %ld %ld %ld\\n",'
            '(long)sizeof(ProresDSPContext),(long)offsetof(ProresDSPContext,idct_permutation_type),'
            '(long)offsetof(ProresDSPContext,idct_permutation),(long)offsetof(ProresDSPContext,idct_put));return 0;}\n')
    try:
        subprocess.run(["gcc", "-x", "c", "-std=c99", "-I", os.path.join(ROOT, "include"), "-", "-o", exe], input=code, text=True, check=True)
        mine = [int(v) for v in subprocess.run([exe], capture_output=True, text=True, check=True).stdout.split()]
    finally:
        if os.path.exists(exe):
            os.remove(exe)
    assert mine == list(out)


def test_hook_fills_what_ff_proresdsp_init_fills(hs, pref):
    """every byte ff_proresdsp_init writes, the hook writes, with the same permutation type and permutation; nothing else"""
    for fill in (0x00, 0xa5):
        a = tables.ProresDSPContext(); b = tables.ProresDSPContext()
        C.memset(C.byref(a), fill, C.sizeof(a)); C.memset(C.byref(b), fill, C.sizeof(b))
        pref.ref_prores_dsp_init(C.byref(a))
        hs.ff_proresdsp_init_cuda(C.byref(b))
        assert a.idct_permutation_type == b.idct_permutation_type == 0                         # FF_IDCT_PERM_NONE
        assert list(a.idct_permutation) == list(b.idct_permutation) == list(range(64))
        assert bool(a.idct_put) and bool(b.idct_put)


def test_header_exports_and_ctypes_agree(built):
    from libav_b200 import _lib
    hdr = open(os.path.join(ROOT, "include", "avdsp_b200.h")).read()
    names = ["ff_prores_idct_put_batch_cuda", "ff_prores_decode_pictures_cuda", "ff_proresdsp_init_cuda"]
    nm = subprocess.run(["nm", "-D", "--defined-only", _lib.LIB_PATH], capture_output=True, text=True, check=True).stdout
    for n in names:
        assert re.search(r"\b%s\(" % n, hdr), n
        assert re.search(r"\bT %s$" % n, nm, re.M), n
        assert n in _lib.PROTOTYPES, n
    W = tables.FFProresPictureWork
    assert C.sizeof(tables.FFProresSlice) == 8
    assert (W.data.offset, W.linesize.offset, W.mb_rows.offset, W.mb_width.offset, W.qmat_luma.offset, W.slices.offset,
            W.n_slices.offset, W.blocks.offset, W.n_blocks.offset, C.sizeof(W)) == (0, 24, 36, 48, 64, 192, 200, 208, 216, 224)
