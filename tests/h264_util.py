"""Picture-level drivers that apply the CPU oracle's per-block H.264 functions in the reference's order -- the
checker for the batched CUDA entry points.  TEST INFRASTRUCTURE."""
import ctypes as C

import numpy as np

from libav_b200 import synth
from oracle.loader import ptr


def at(a, off):
    return C.c_void_p(a.ctypes.data + int(off))


def block_offsets(ls, uvls):
    """frame-MB block_offset[] (libavcodec/h264_slice.c:486-493) for luma 0..15 and chroma 16..19 / 32..35"""
    bo = np.zeros(48, dtype=np.int32)
    for i in range(16):
        bo[i] = 4 * ((i & 1) + 2 * ((i >> 2) & 1)) + 4 * (((i >> 1) & 1) + 2 * (i >> 3)) * ls
    for i in range(4):
        bo[16 + i] = bo[32 + i] = 4 * (i & 1) + 4 * ((i >> 1) & 1) * uvls
    return bo


def block_offsets_422(uvls):
    """block_offset[] entries ff_h264_idct_add8_422 reads: chroma blocks 16..19 / 32..35 (upper 8 rows) and 24..27 / 40..43
    (lower 8 rows) of an 8x16 chroma macroblock"""
    bo = np.zeros(48, dtype=np.int32)
    for i in range(4):
        bo[16 + i] = bo[32 + i] = 4 * (i & 1) + 4 * ((i >> 1) & 1) * uvls
        bo[24 + i] = bo[40 + i] = 4 * (i & 1) + (8 + 4 * ((i >> 1) & 1)) * uvls
    return bo


def scan8(i):
    plane, k = i >> 4, i & 15
    return 4 + (k & 1) + 2 * ((k >> 2) & 1) + 8 * (1 + ((k >> 1) & 1) + 2 * (k >> 3) + 5 * plane)


def residual_422(seed):
    """coefficients (48 x 16 int16, sl->mb layout) and non_zero_count_cache for one 4:2:2 macroblock's chroma: per 4x4 block
    nothing / DC only with nnz 0 (the dc_add branch) / full block, like the decoder leaves them after the chroma DC transform"""
    rng = np.random.default_rng(1000 + seed)
    coeffs = np.zeros((48, 16), np.int16)
    nnzc = np.zeros(120, np.uint8)
    for plane in (1, 2):
        for k in range(8):
            i = 16 * plane + k                        # coefficient block
            e = i + 4 if k >= 4 else i                # cache / offset entry
            kind = int(rng.integers(0, 3))
            if kind == 1:
                coeffs[i, 0] = rng.integers(-2000, 2000)
            elif kind == 2:
                coeffs[i] = rng.integers(-600, 600, size=16)
                nnzc[scan8(e)] = rng.integers(1, 16)
    return coeffs, nnzc


def oracle_residual(o, rec, coeffs, nnzc, y, cb, cr):
    ls, uvls = y.strides[0], cb.strides[0]
    bo = block_offsets(ls, uvls)
    for m in range(rec.shape[0]):
        r = rec[m]
        blk, nz = coeffs[m], nnzc[m]
        if r["luma_mode"] < 3:
            o.h264_idct_mb(int(r["luma_mode"]), at(y, r["luma_off"]), None, ptr(bo), ptr(blk), ls, ptr(nz))
        if r["chroma"]:
            d2 = (C.c_void_p * 2)(cb.ctypes.data + int(r["chroma_off"]), cr.ctypes.data + int(r["chroma_off"]))
            o.h264_idct_mb(3, None, d2, ptr(bo), ptr(blk), uvls, ptr(nz))


def padded(plane, pad):
    p = np.pad(plane, pad, mode="edge")
    return p, p[pad:-pad, pad:-pad]


def _window(base, sy, sx, h, w):
    """base[sy:sy + h, sx:sx + w], refusing a window the padding does not hold (a negative start would wrap around in numpy)"""
    assert sy >= 0 and sx >= 0 and sy + h <= base.shape[0] and sx + w <= base.shape[1], "oracle_mc: pad too small for this vector"
    return base[sy:sy + h, sx:sx + w]


def oracle_mc(o, rec, refs, y, cb, cr, pad=48):
    """refs: list of (y, cb, cr) planes; edge replication is emulated by padding the reference planes by `pad` samples, which
    must cover the farthest vector of `rec` (asserted per window)."""
    pr = []
    for (ry, rcb, rcr) in refs:
        pr.append((padded(ry, pad)[1], padded(rcb, pad)[1], padded(rcr, pad)[1]))
    sizes = {16: 0, 8: 1, 4: 2, 2: 3}
    for r in rec:
        ry, rcb, rcr = pr[int(r["ref"])]
        mx, my = int(r["mvx"]) + 4 * int(r["x"]), int(r["mvy"]) + 4 * int(r["y"])
        w, h, avg = int(r["w"]), int(r["h"]), int(r["avg"])
        mc = (mx & 3) + 4 * (my & 3)
        # the reference's qpel functions are square: non-square partitions are two calls (h264_mb.c:248-250)
        n = min(w, h)
        for (ox, oy) in [(a, b) for b in range(0, h, n) for a in range(0, w, n)]:
            src = at(ry, ((my >> 2) + oy) * ry.strides[0] + (mx >> 2) + ox)
            dst = at(y, (int(r["y"]) + oy) * y.strides[0] + int(r["x"]) + ox)
            # qpel needs one stride for src and dst: copy the source window into a dst-stride scratch
            win = np.zeros((n + 5, y.strides[0]), np.uint8)
            sy, sx = (my >> 2) + oy - 2, (mx >> 2) + ox - 2
            base = ry.base if ry.base is not None else ry
            win[:, :n + 5] = _window(base, sy + pad, sx + pad, n + 5, n + 5)
            o.h264_qpel(avg, sizes[n], mc, dst, at(win, 2 * win.strides[0] + 2), y.strides[0])
        cw, chh = w // 2, h // 2
        for (pl, rp) in ((cb, rcb), (cr, rcr)):
            base = rp.base if rp.base is not None else rp
            sy, sx = (my >> 3), (mx >> 3)
            win = np.zeros((chh + 1, pl.strides[0]), np.uint8)
            win[:, :cw + 1] = _window(base, sy + pad, sx + pad, chh + 1, cw + 1)
            dst = at(pl, (int(r["y"]) // 2) * pl.strides[0] + int(r["x"]) // 2)
            o.h264_chroma(avg, {8: 0, 4: 1, 2: 2}[cw], dst, ptr(win), pl.strides[0], chh, mx & 7, my & 7)


def oracle_deblock(o, rec, mb_w, mb_h, y, cb, cr):
    ls, uvls = y.strides[0], cb.strides[0]
    for m in range(mb_w * mb_h):
        r = rec[m]
        mbx, mby = m % mb_w, m // mb_w
        for d in (0, 1):
            for e in range(4):
                a, b = int(r["alpha"][d, e]), int(r["beta"][d, e])
                if a and b:
                    off = (mby * 16 + (4 * e if d else 0)) * ls + mbx * 16 + (0 if d else 4 * e)
                    intra = (int(r["intra"][d]) >> e) & 1
                    which = (1 if d == 0 else 0) + (2 if intra else 0)
                    tc = np.ascontiguousarray(r["tc0"][d, e])
                    o.h264_loop_filter(which, at(y, off), ls, a, b, ptr(tc))
                if not (e & 1):
                    ce = e >> 1
                    for p, pl in enumerate((cb, cr)):
                        a, b = int(r["calpha"][p, d, ce]), int(r["cbeta"][p, d, ce])
                        if a and b:
                            off = (mby * 8 + (4 * ce if d else 0)) * uvls + mbx * 8 + (0 if d else 4 * ce)
                            intra = (int(r["cintra"][p, d]) >> ce) & 1
                            which = 4 + (1 if d == 0 else 0) + (2 if intra else 0)
                            tc = np.ascontiguousarray(r["ctc0"][p, d, ce])
                            o.h264_loop_filter(which, at(pl, off), uvls, a, b, ptr(tc))


def oracle_weight(o, rec, plane, src=None):
    widx = {16: 0, 8: 1, 4: 2, 2: 3}
    st = plane.strides[0]
    for r in rec:
        if src is None:
            o.h264_weight(widx[int(r["w"])], at(plane, r["off"]), st, int(r["h"]), int(r["log2_denom"]), int(r["weight"]), int(r["offset"]))
        else:
            o.h264_biweight(widx[int(r["w"])], at(plane, r["off"]), at(src, r["off"]), st, int(r["h"]), int(r["log2_denom"]),
                            int(r["weight"]), int(r["weight_src"]), int(r["offset"]))


def oracle_intra(o, rec, coeffs, nnzc, mb_w, mb_h, y, cb, cr):
    """hl_decode_mb() for intra macroblocks (h264_mb.c:607-731, h264_mb_template.c:158-197): prediction and residual block
    by block through the oracle's H264PredContext / H264DSPContext entries."""
    ls, uvls = y.strides[0], cb.strides[0]
    for m in range(mb_w * mb_h):
        r = rec[m]
        kind = int(r["kind"])
        if kind == 0:
            continue
        mbx, mby = m % mb_w, m // mb_w
        mb = coeffs[m]
        org = mby * 16 * ls + mbx * 16
        corg = mby * 8 * uvls + mbx * 8
        if kind in (1, 2):
            for i in range(0, 16, 1 if kind == 1 else 4):
                bx, by = (i & 1) + 2 * ((i >> 2) & 1), ((i >> 1) & 1) + 2 * (i >> 3)
                off = org + 4 * by * ls + 4 * bx
                mode = int(r["mode4"][i])
                nnz = int(nnzc[m, synth.scan8(i)])
                blk = mb[16 * i:]
                if kind == 1:
                    tr_ok = (int(r["topright"]) << i) & 0x8000
                    if mode in (3, 7) and not tr_ok:
                        tr = np.full(4, y[mby * 16 + 4 * by - 1, mbx * 16 + 4 * bx + 3], np.uint8)
                        o.h264_pred(0, mode, at(y, off), ptr(tr), 0, 0, ls)
                    else:
                        o.h264_pred(0, mode, at(y, off), at(y, off + 4 - ls), 0, 0, ls)
                    if nnz:
                        o.h264_idct(2 if (nnz == 1 and blk[0]) else 0, at(y, off), ptr(blk), ls)
                else:
                    o.h264_pred(1, mode, at(y, off), None, (int(r["topleft"]) << i) & 0x8000, (int(r["topright"]) << i) & 0x4000, ls)
                    if nnz:
                        o.h264_idct(3 if (nnz == 1 and blk[0]) else 1, at(y, off), ptr(blk), ls)
        else:
            o.h264_pred(3, int(r["mode16"]), at(y, org), None, 0, 0, ls)
            bo = np.array([4 * ((i & 1) + 2 * ((i >> 2) & 1)) + 4 * (((i >> 1) & 1) + 2 * (i >> 3)) * ls for i in range(16)] + [0] * 32, np.int32)
            o.h264_idct_mb(1, at(y, org), None, ptr(bo), ptr(mb), ls, ptr(nnzc[m]))
        for pl in (cb, cr):
            o.h264_pred(2, int(r["chroma_mode"]), at(pl, corg), None, 0, 0, uvls)
        if r["chroma_residual"]:
            bo = np.zeros(48, np.int32)
            for k in range(4):
                bo[16 + k] = bo[32 + k] = 4 * (k & 1) + 4 * (k >> 1) * uvls
            dst2 = (C.c_void_p * 2)(at(cb, corg), at(cr, corg))
            o.h264_idct_mb(3, None, dst2, ptr(bo), ptr(mb), uvls, ptr(nnzc[m]))
