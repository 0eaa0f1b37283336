"""The product's H264DSPContext loop-filter slots under the reference's OWN deblocking driver: h264_loopfilter.c (ff_h264_filter_mb_fast ->
ff_h264_filter_mb), compiled unmodified into oracle/_ref, walks a picture in raster order like loop_filter() and calls the table's
entries on the real planes -- once with the reference's C functions, once with the table ff_h264dsp_init_cuda() filled.  Same bytes or
the slots are not a drop-in.  At 9 / 10 bit the planes hold uint16 samples and the side information is in the decoder's QP' scale.  Shared by
the host simulation (CPU) and the product library (GPU).  TEST INFRASTRUCTURE."""
import ctypes as C

import numpy as np

from libav_b200 import synth
from oracle.loader import ptr

CASES = [dict(seed=1), dict(seed=2, bipred=True), dict(seed=3, t8x8=1, cabac=1), dict(seed=5, t8x8=1, cabac=0, bipred=True, mode=2, n_slices=5),
         dict(seed=6, mode=2, n_slices=7, p_intra=0.4), dict(seed=8, cb_off=-3, cr_off=5, bipred=True)]


def run(refo, table, d, planes):
    """table NULL: the reference's own C functions for d's bit depth"""
    y, cb, cr = [p.copy() for p in planes]
    args = (table, ptr(y), ptr(cb), ptr(cr), y.strides[0], cb.strides[0], d["mb_w"], d["mb_h"], ptr(d["mb_type"]), ptr(d["qscale"]), ptr(d["nnz"]),
            ptr(d["cbp"]), ptr(d["slice_table"]), ptr(d["mv0"]), ptr(d["mv1"]), ptr(d["ref0"]), ptr(d["ref1"]), ptr(d["slice_params"]), d["n_slices"],
            ptr(d["chroma_qp_table"]), d["cabac"], d["t8x8"])
    bits = d.get("bit_depth", 8)
    rc = refo.h264_deblock_picture_with(*args) if bits == 8 else refo.h264_deblock_picture_with_hbd(bits, *args)
    assert rc == 0
    return y, cb, cr


def check(refo, lib, sizes=((6, 4), (2, 5), (1, 1)), bits=8):
    from libav_b200 import tables
    t = tables.H264DSPContext()
    lib.ff_h264dsp_init_cuda(C.byref(t), bits, 1)
    n = changed = 0
    sc, dt = 1 << (bits - 8), np.uint8 if bits == 8 else np.uint16
    for case in CASES:
        for (mw, mh) in sizes:
            d = synth.h264_deblock_info(mw, mh, bit_depth=bits, **case)
            rng = np.random.default_rng(case["seed"] + mw)
            base = rng.integers(40, 200)
            planes = [(np.clip(base + rng.integers(-12, 13, size=(16 * mh, 16 * mw + 16)), 0, 255) * sc).astype(dt),
                      (np.clip(base + rng.integers(-12, 13, size=(8 * mh, 8 * mw + 8)), 0, 255) * sc).astype(dt),
                      (np.clip(base + rng.integers(-12, 13, size=(8 * mh, 8 * mw + 8)), 0, 255) * sc).astype(dt)]
            want = run(refo, None, d, planes)
            got = run(refo, C.byref(t), d, planes)
            for a, b in zip(got, want):
                assert np.array_equal(a, b), (case, mw, mh, np.argwhere(a != b)[:4].tolist())
            changed += not np.array_equal(want[0], planes[0])
            n += 1
    assert changed > n // 2                     # the pictures are smooth enough for the filters to fire
    return n
