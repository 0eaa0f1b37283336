"""9 / 10-bit (and 4:2:2) pictures for the batched H.264 calls (libav_b200/csrc/h264_hbd_batch.cu): generators and the picture-level
checker that applies the CPU oracle's per-block functions (the reference's own BIT_DEPTH > 8 instances) in the reference's order.
TEST INFRASTRUCTURE."""
import ctypes as C

import numpy as np

from libav_b200 import synth
from oracle.loader import ptr
from h264_util import at, scan8


def picture(mb_w, mb_h, bits, c422, seed):
    rng = np.random.default_rng(seed)
    w, h = 16 * mb_w, 16 * mb_h
    ch = h if c422 else h // 2
    dt = np.uint8 if bits == 8 else np.uint16          # (bits 8: the 8-bit 4:2:2 pictures the generic kernels also take)
    return (rng.integers(0, 1 << bits, (h, w)).astype(dt), rng.integers(0, 1 << bits, (ch, w // 2)).astype(dt),
            rng.integers(0, 1 << bits, (ch, w // 2)).astype(dt))


def block_offsets(ls, uvls, c422, sb=2):
    """block_offset[] in BYTES (h264_slice.c:486-493; sb = bytes per sample: pixel_shift 1 for 16-bit samples): luma 0..15, chroma 16.. / 32..
    (4:2:2: the entries ff_h264_idct_add8_422 reads, 16..19 and 24..27 per plane)"""
    bo = np.zeros(48, dtype=np.int32)
    for i in range(16):
        bo[i] = sb * 4 * ((i & 1) + 2 * ((i >> 2) & 1)) + 4 * (((i >> 1) & 1) + 2 * (i >> 3)) * ls
    for i in range(4):
        bo[16 + i] = bo[32 + i] = sb * 4 * (i & 1) + 4 * ((i >> 1) & 1) * uvls
        if c422:
            bo[24 + i] = bo[40 + i] = sb * 4 * (i & 1) + (8 + 4 * ((i >> 1) & 1)) * uvls
    return bo


def residual_work(mb_w, mb_h, bits, c422, y, cb, seed):
    """records (byte offsets for these planes), int32 coefficients (n, 768), nnzc (n, 120)"""
    rng = np.random.default_rng(seed)
    n = mb_w * mb_h
    rec = np.zeros(n, dtype=synth.RESIDUAL_DT)
    mbx, mby = np.arange(n) % mb_w, np.arange(n) // mb_w
    sb = y.itemsize
    rec["luma_off"] = mby * 16 * y.strides[0] + mbx * 16 * sb
    rec["chroma_off"] = mby * (16 if c422 else 8) * cb.strides[0] + mbx * 8 * sb
    rec["luma_mode"] = rng.choice(np.array([0, 1, 2, 3], dtype=np.uint8), size=n)
    rec["chroma"] = rng.integers(0, 2, size=n)
    coeffs = np.zeros((n, 768), dtype=np.int16 if bits == 8 else np.int32)
    nnzc = np.zeros((n, 120), dtype=np.uint8)
    sc = 1 << (bits - 8)
    chroma_blocks = [16, 17, 18, 19, 32, 33, 34, 35] + ([20, 21, 22, 23, 36, 37, 38, 39] if c422 else [])
    for m in range(n):
        mode = int(rec["luma_mode"][m])
        blocks = list(range(0, 16, 4)) if mode == 2 else list(range(16))
        for i in blocks + chroma_blocks:
            sz = 64 if (mode == 2 and i < 16) else 16
            kind = rng.integers(0, 4) if rng.random() < 0.75 else 0       # 0 none, 1 dc only (nnz 0), 2 dc (nnz 1), 3 full
            if kind == 0:
                continue
            e = i + 4 if (i & 15) >= 4 and i >= 16 else i                  # 4:2:2 lower half: nnz lives at scan8[i + 4]
            if kind in (1, 2):
                coeffs[m, 16 * i] = rng.integers(-2000 * sc, 2000 * sc)
                nnzc[m, scan8(e)] = 0 if kind == 1 else 1
            else:
                coeffs[m, 16 * i:16 * i + sz] = rng.integers(-300 * sc, 300 * sc, size=sz)
                nnzc[m, scan8(e)] = rng.integers(2, 17)
    return rec, coeffs, nnzc


def oracle_residual(o, bits, c422, rec, coeffs, nnzc, y, cb, cr):
    ls, uvls = y.strides[0], cb.strides[0]
    bo = block_offsets(ls, uvls, c422, y.itemsize)
    idct_mb = (lambda which, d, d2, blk, st, nz: o.h264_idct_mb(which, d, d2, ptr(bo), ptr(blk), st, ptr(nz))) if bits == 8 else \
              (lambda which, d, d2, blk, st, nz: o.h264_hbd_idct_mb(bits, which, d, d2, ptr(bo), ptr(blk), st, ptr(nz)))
    for m in range(rec.shape[0]):
        r = rec[m]
        blk, nz = coeffs[m], nnzc[m]
        if r["luma_mode"] < 3:
            idct_mb(int(r["luma_mode"]), at(y, r["luma_off"]), None, blk, ls, nz)
        if r["chroma"]:
            d2 = (C.c_void_p * 2)(cb.ctypes.data + int(r["chroma_off"]), cr.ctypes.data + int(r["chroma_off"]))
            idct_mb(4 if c422 else 3, None, d2, blk, uvls, nz)


def oracle_mc(o, bits, c422, rec, refs, y, cb, cr, pw=None, ph=None):
    """refs: list of (y, cb, cr) planes (uint16 above 8 bit); emulated_edge_mc = the reference planes cropped to pw x ph (default: the
    destination's size) and edge-replicated as far as the farthest vector of `rec` reaches (h264_edge_cases.mc_pad).  The records run
    in put-then-avg order, as the batch call promises whatever their order in `rec`."""
    import h264_edge_cases as ec
    pw, ph = pw or y.shape[1], ph or y.shape[0]
    cph = ph if c422 else ph >> 1
    pad = ec.mc_pad(rec, pw, ph)                      # (also enough for 4:2:2 chroma: its rows reach no farther than the luma taps)
    pr = [(np.pad(r[0][:ph, :pw], pad, mode="edge"), np.pad(r[1][:cph, :pw >> 1], pad, mode="edge"), np.pad(r[2][:cph, :pw >> 1], pad, mode="edge"))
          for r in refs]
    rec = np.concatenate([rec[rec["avg"] == 0], rec[rec["avg"] != 0]])
    sizes = {16: 0, 8: 1, 4: 2, 2: 3}
    sb, dt = y.itemsize, y.dtype
    qpel = (lambda avg, sidx, mc, dst, src, st: o.h264_qpel(avg, sidx, mc, dst, src, st)) if bits == 8 else \
           (lambda avg, sidx, mc, dst, src, st: o.h264_hbd_qpel(bits, avg, sidx, mc, dst, src, st))
    chroma = (lambda avg, widx, dst, src, st, hh_, fx, fy: o.h264_chroma(avg, widx, dst, src, st, hh_, fx, fy)) if bits == 8 else \
             (lambda avg, widx, dst, src, st, hh_, fx, fy: o.h264_hbd_chroma(bits, avg, widx, dst, src, st, hh_, fx, fy))
    for r in rec:
        ry, rcb, rcr = pr[int(r["ref"])]
        mx, my = int(r["mvx"]) + 4 * int(r["x"]), int(r["mvy"]) + 4 * int(r["y"])
        w, h, avg = int(r["w"]), int(r["h"]), int(r["avg"])
        mc = (mx & 3) + 4 * (my & 3)
        n = min(w, h)
        for (ox, oy) in [(a, b) for b in range(0, h, n) for a in range(0, w, n)]:     # square calls (h264_mb.c:248-250)
            dst = at(y, (int(r["y"]) + oy) * y.strides[0] + sb * (int(r["x"]) + ox))
            win = np.zeros((n + 5, y.strides[0] // sb), dt)                             # source window at the destination's pitch
            sy, sx = (my >> 2) + oy - 2 + pad, (mx >> 2) + ox - 2 + pad
            win[:, :n + 5] = ry[sy:sy + n + 5, sx:sx + n + 5]
            qpel(avg, sizes[n], mc, dst, at(win, 2 * win.strides[0] + 2 * sb), y.strides[0])
        cw, chh = w // 2, (h if c422 else h // 2)
        sy, sx = ((my >> 2) if c422 else (my >> 3)) + pad, (mx >> 3) + pad
        fy = ((my << 1) & 7) if c422 else (my & 7)
        for (pl, rp) in ((cb, rcb), (cr, rcr)):
            win = np.zeros((chh + 1, pl.strides[0] // sb), dt)
            win[:, :cw + 1] = rp[sy:sy + chh + 1, sx:sx + cw + 1]
            dst = at(pl, (int(r["y"]) if c422 else int(r["y"]) // 2) * pl.strides[0] + sb * (int(r["x"]) // 2))
            chroma(avg, {8: 0, 4: 1, 2: 2}[cw], dst, ptr(win), pl.strides[0], chh, mx & 7, fy)


def oracle_deblock(o, bits, rec, mb_w, mb_h, y, cb, cr):
    ls, uvls = y.strides[0], cb.strides[0]
    for m in range(mb_w * mb_h):
        r = rec[m]
        mbx, mby = m % mb_w, m // mb_w
        for d in (0, 1):
            for e in range(4):
                a, b = int(r["alpha"][d, e]), int(r["beta"][d, e])
                if a and b:
                    off = (mby * 16 + (4 * e if d else 0)) * ls + 2 * (mbx * 16 + (0 if d else 4 * e))
                    intra = (int(r["intra"][d]) >> e) & 1
                    tc = np.ascontiguousarray(r["tc0"][d, e])
                    o.h264_hbd_loop_filter(bits, (1 if d == 0 else 0) + (2 if intra else 0), at(y, off), ls, a, b, ptr(tc))
                if not (e & 1):
                    ce = e >> 1
                    for p, pl in enumerate((cb, cr)):
                        a, b = int(r["calpha"][p, d, ce]), int(r["cbeta"][p, d, ce])
                        if a and b:
                            off = (mby * 8 + (4 * ce if d else 0)) * uvls + 2 * (mbx * 8 + (0 if d else 4 * ce))
                            intra = (int(r["cintra"][p, d]) >> ce) & 1
                            tc = np.ascontiguousarray(r["ctc0"][p, d, ce])
                            o.h264_hbd_loop_filter(bits, 4 + (1 if d == 0 else 0) + (2 if intra else 0), at(pl, off), uvls, a, b, ptr(tc))


def smooth_picture(mb_w, mb_h, bits, seed):
    """smooth content + noise so that a large share of the edges really gets filtered"""
    rng = np.random.default_rng(seed)
    sc = 1 << (bits - 8)

    def plane(shape):
        base = rng.integers(40, 200, size=(shape[0] // 8 + 1, shape[1] // 8 + 1))
        up = np.kron(base, np.ones((8, 8), dtype=np.int64))[:shape[0], :shape[1]]
        return np.clip(sc * (up + rng.integers(-6, 7, size=shape)) + rng.integers(0, sc, size=shape), 0, (1 << bits) - 1).astype(np.uint16)
    return plane((16 * mb_h, 16 * mb_w)), plane((8 * mb_h, 8 * mb_w)), plane((8 * mb_h, 8 * mb_w))


# ---- 4:2:2 deblocking (8 / 9 / 10 bit): the 52-byte record of the four horizontal chroma edges ------------------------------------------
CHROMA422_DT = np.dtype([("alpha", "u1", (2, 4)), ("beta", "u1", (2, 4)), ("tc0", "i1", (2, 4, 4)), ("intra", "u1", (2,)), ("pad", "u1", (2,))])
assert CHROMA422_DT.itemsize == 52


def deblock422_work(mb_w, mb_h, seed, slices=1):
    """(104-byte records, 52-byte records) with random per-edge parameters in the ranges of the reference's tables; picture- and slice-boundary
    edges carry alpha 0 like synth.h264_deblock_work makes them"""
    rec = synth.h264_deblock_work(mb_w, mb_h, seed=seed, slices=slices)
    rng = np.random.default_rng(1000 + seed)
    n = mb_w * mb_h
    ext = np.zeros(n, CHROMA422_DT)
    ext["alpha"] = rng.integers(0, 120, (n, 2, 4)); ext["beta"] = rng.integers(0, 19, (n, 2, 4))
    ext["tc0"] = rng.integers(0, 11, (n, 2, 4, 4)); ext["intra"] = rng.integers(0, 2, (n, 2))       # only edge 0 may be intra
    ext["alpha"][:, :, 0] = np.where(rec["alpha"][:, 1, 0][:, None] == 0, 0, ext["alpha"][:, :, 0])   # top edge off where the luma one is (boundaries)
    rec["calpha"][:, :, 1, :] = 0                                                                      # not read in 4:2:2
    return rec, ext


def oracle_deblock422(o, bits, rec, ext, mb_w, mb_h, y, cb, cr):
    """luma from the 104-byte record; chroma: vertical edges = h_loop_filter_chroma422 (16 lines, which 12 / 13), horizontal edges = the four
    v_loop_filter_chroma calls of h264_loopfilter.c:693-700 (which 4 / 6), in the reference's order: per direction, edge by edge"""
    ls, uvls, sb = y.strides[0], cb.strides[0], (1 if bits == 8 else 2)
    lf = (lambda which, p, st, a, b, tc: o.h264_loop_filter(which, p, st, a, b, tc)) if bits == 8 else \
         (lambda which, p, st, a, b, tc: o.h264_hbd_loop_filter(bits, which, p, st, a, b, tc))
    for m in range(mb_w * mb_h):
        r, x = rec[m], ext[m]
        mbx, mby = m % mb_w, m // mb_w
        for d in (0, 1):
            for e in range(4):
                a, b = int(r["alpha"][d, e]), int(r["beta"][d, e])
                if a and b:
                    off = (mby * 16 + (4 * e if d else 0)) * ls + sb * (mbx * 16 + (0 if d else 4 * e))
                    intra = (int(r["intra"][d]) >> e) & 1
                    lf((1 if d == 0 else 0) + (2 if intra else 0), at(y, off), ls, a, b, ptr(np.ascontiguousarray(r["tc0"][d, e])))
                for p, pl in enumerate((cb, cr)):
                    if d == 0 and not (e & 1):
                        ce = e >> 1
                        a, b = int(r["calpha"][p, 0, ce]), int(r["cbeta"][p, 0, ce])
                        if a and b:
                            off = mby * 16 * uvls + sb * (mbx * 8 + 4 * ce)
                            intra = (int(r["cintra"][p, 0]) >> ce) & 1
                            lf(13 if intra else 12, at(pl, off), uvls, a, b, ptr(np.ascontiguousarray(r["ctc0"][p, 0, ce])))
                    elif d == 1:
                        a, b = int(x["alpha"][p, e]), int(x["beta"][p, e])
                        if a and b:
                            off = (mby * 16 + 4 * e) * uvls + sb * mbx * 8
                            intra = (int(x["intra"][p]) >> e) & 1
                            lf(6 if intra else 4, at(pl, off), uvls, a, b, ptr(np.ascontiguousarray(x["tc0"][p, e])))


def smooth_picture422(mb_w, mb_h, bits, seed):
    rng = np.random.default_rng(seed)
    sc = 1 << (bits - 8)

    def plane(shape):
        base = rng.integers(40, 200, size=(shape[0] // 8 + 1, shape[1] // 8 + 1))
        up = np.kron(base, np.ones((8, 8), dtype=np.int64))[:shape[0], :shape[1]]
        v = np.clip(sc * (up + rng.integers(-6, 7, size=shape)) + rng.integers(0, sc, size=shape), 0, (1 << bits) - 1)
        return v.astype(np.uint8 if bits == 8 else np.uint16)
    return plane((16 * mb_h, 16 * mb_w)), plane((16 * mb_h, 8 * mb_w)), plane((16 * mb_h, 8 * mb_w))


# ---- weighted prediction and DC transforms at 9 / 10 bit ------------------------------------------------------------------------------------
WIDX = {16: 0, 8: 1, 4: 2, 2: 3}


def oracle_weight(o, bits, rec, plane, src=None):
    """the reference's weight_h264_pixels / biweight_h264_pixels at `bits` over `rec` (byte offsets) in place on `plane`"""
    st = plane.strides[0]
    for r in rec:
        if src is not None:
            o.h264_hbd_biweight(bits, WIDX[int(r["w"])], at(plane, r["off"]), at(src, r["off"]), st, int(r["h"]), int(r["log2_denom"]), int(r["weight"]),
                                int(r["weight_src"]), int(r["offset"]))
        else:
            o.h264_hbd_weight(bits, WIDX[int(r["w"])], at(plane, r["off"]), st, int(r["h"]), int(r["log2_denom"]), int(r["weight"]), int(r["offset"]))


def oracle_dc(o, bits, c422, recs, coeffs, luma_dc):
    """the reference's luma / chroma (4:2:2: chroma422) DC dequantisation in place on the int32 arena `coeffs` (n, 768)"""
    for m in range(recs.shape[0]):
        if recs["luma_qmul"][m]:
            o.h264_hbd_dc_dequant(bits, 0, at(coeffs, m * 768 * 4), ptr(luma_dc[m].copy()), int(recs["luma_qmul"][m]))
        for pl in range(2):
            if recs["chroma_qmul"][m, pl]:
                o.h264_hbd_dc_dequant(bits, 2 if c422 else 1, at(coeffs, (m * 768 + 256 * (pl + 1)) * 4), None, int(recs["chroma_qmul"][m, pl]))


def weight_dc_cases(run_weight, run_dc, o, bits):
    """run_weight(bits, rec, plane, src | None) -> plane after ff_h264_weight_batch_hbd_cuda; run_dc(c422, recs, coeffs, luma_dc) -> coeffs after
    ff_h264_dc_dequant_batch_hbd_cuda; both against the oracle's BIT_DEPTH > 8 functions"""
    rng = np.random.default_rng(bits)
    for bi in (0, 1):
        plane = rng.integers(0, 1 << bits, size=(128, 256)).astype(np.uint16)
        src = rng.integers(0, 1 << bits, size=(128, 256)).astype(np.uint16)
        recs = []
        for by in range(0, 128, 16):
            for bx in range(0, 256, 16):
                w = int(rng.choice([16, 8, 4, 2]))
                recs.append(((by * 256 + bx) * 2, w, int(rng.choice([2, 4, 8, 16])), int(rng.integers(0, 8)), 0, int(rng.integers(-128, 128)),
                             int(rng.integers(-128, 128)), int(rng.integers(-128, 128)), 0))
        rec = np.array(recs, dtype=synth.WEIGHT_DT)
        want = plane.copy()
        oracle_weight(o, bits, rec, want, src if bi else None)
        got = run_weight(bits, rec, plane.copy(), src if bi else None)
        assert not np.array_equal(want, plane) and np.array_equal(got, want), ("weight", bits, bi, np.argwhere(got != want)[:4].tolist())
    DC_DT = np.dtype([("luma_qmul", "<u4"), ("chroma_qmul", "<u4", (2,))])
    for c422 in (0, 1):
        n = 300
        recs = np.zeros(n, DC_DT)
        recs["luma_qmul"] = np.where(rng.random(n) < 0.6, rng.integers(16, 4000, n), 0)
        recs["chroma_qmul"] = np.where(rng.random((n, 2)) < 0.6, rng.integers(16, 4000, (n, 2)), 0)
        sc = 1 << (bits - 8)
        coeffs = rng.integers(-300 * sc, 300 * sc, size=(n, 768)).astype(np.int32)
        luma_dc = rng.integers(-2000 * sc, 2000 * sc, size=(n, 16)).astype(np.int32)
        want = coeffs.copy()
        oracle_dc(o, bits, c422, recs, want, luma_dc)
        got = run_dc(c422, recs, coeffs.copy(), luma_dc)
        assert not np.array_equal(want, coeffs) and np.array_equal(got, want), ("dc", bits, c422, np.argwhere(got != want)[:4].tolist())


# ---- intra reconstruction at 9 / 10 bit ---------------------------------------------------------------------------------------------------
def oracle_intra(o, bits, rec, coeffs, nnzc, mb_w, mb_h, y, cb, cr, c422=0):
    """hl_decode_mb() for intra macroblocks (h264_mb.c:607-731, h264_mb_template.c:158-197) through the oracle's H264PredContext / H264DSPContext
    entries of that bit depth, block by block (tests/h264_util.py::oracle_intra generalised: 16-bit samples above 8 bit, strides and offsets in
    bytes; c422: the 8 x 16 chroma predictors and h264_idct_add8_422)"""
    ls, uvls, sb = y.strides[0], cb.strides[0], y.itemsize
    if bits == 8:
        pred = lambda tab, mode, src, tr, tl, trf, st: o.h264_pred(tab, mode, src, tr, tl, trf, st)
        idct = lambda which, d, blk, st: o.h264_idct(which, d, blk, st)
        idct_mb = lambda which, d, d2, bo, blk, st, nz: o.h264_idct_mb(which, d, d2, bo, blk, st, nz)
    else:
        pred = lambda tab, mode, src, tr, tl, trf, st: o.h264_hbd_pred(bits, tab, mode, src, tr, tl, trf, st)
        idct = lambda which, d, blk, st: o.h264_hbd_idct(bits, which, d, blk, st)
        idct_mb = lambda which, d, d2, bo, blk, st, nz: o.h264_hbd_idct_mb(bits, which, d, d2, bo, blk, st, nz)
    bo = block_offsets(ls, uvls, c422, sb)
    for m in range(mb_w * mb_h):
        r = rec[m]
        kind = int(r["kind"])
        if kind == 0:
            continue
        mbx, mby = m % mb_w, m // mb_w
        mb = coeffs[m]
        org = mby * 16 * ls + mbx * 16 * sb
        corg = mby * (16 if c422 else 8) * uvls + mbx * 8 * sb
        if kind in (1, 2):
            for i in range(0, 16, 1 if kind == 1 else 4):
                bx, by = (i & 1) + 2 * ((i >> 2) & 1), ((i >> 1) & 1) + 2 * (i >> 3)
                off = org + 4 * by * ls + 4 * sb * bx
                mode = int(r["mode4"][i])
                nnz = int(nnzc[m, synth.scan8(i)])
                blk = mb[16 * i:]
                if kind == 1:
                    tr_ok = (int(r["topright"]) << i) & 0x8000
                    if mode in (3, 7) and not tr_ok:
                        tr = np.full(4, y[mby * 16 + 4 * by - 1, mbx * 16 + 4 * bx + 3], y.dtype)
                        pred(0, mode, at(y, off), ptr(tr), 0, 0, ls)
                    else:
                        pred(0, mode, at(y, off), at(y, off + 4 * sb - ls), 0, 0, ls)
                    if nnz:
                        idct(2 if (nnz == 1 and blk[0]) else 0, at(y, off), ptr(blk), ls)
                else:
                    pred(1, mode, at(y, off), None, (int(r["topleft"]) << i) & 0x8000, (int(r["topright"]) << i) & 0x4000, ls)
                    if nnz:
                        idct(3 if (nnz == 1 and blk[0]) else 1, at(y, off), ptr(blk), ls)
        else:
            pred(3, int(r["mode16"]), at(y, org), None, 0, 0, ls)
            idct_mb(1, at(y, org), None, ptr(bo), ptr(mb), ls, ptr(nnzc[m]))
        for pl in (cb, cr):
            if c422:
                o.h264_pred422(bits, int(r["chroma_mode"]), at(pl, corg), uvls)
            else:
                pred(2, int(r["chroma_mode"]), at(pl, corg), None, 0, 0, uvls)
        if r["chroma_residual"]:
            dst2 = (C.c_void_p * 2)(cb.ctypes.data + corg, cr.ctypes.data + corg)
            idct_mb(4 if c422 else 3, None, dst2, ptr(bo), ptr(mb), uvls, ptr(nnzc[m]))


def intra_work(mb_w, mb_h, bits, seed, p_intra=1.0, c422=0):
    """synth.h264_intra_work at this bit depth (int32 coefficients above 8 bit); c422: the lower four chroma blocks of each plane as well
    (coefficients at block 20..23 / 36..39, their non_zero_count at scan8[i + 4] like h264_idct_add8_422 reads them)"""
    rec, coeffs, nnzc = synth.h264_intra_work(mb_w, mb_h, seed=seed, p_intra=p_intra)
    if c422:
        rng = np.random.default_rng(seed + 77)
        for m in np.nonzero(rec["chroma_residual"])[0]:
            for i in (20, 21, 22, 23, 36, 37, 38, 39):
                u = rng.random()
                if u < 0.3:
                    continue
                if u < 0.5:
                    coeffs[m, 16 * i] = rng.integers(-800, 801) or 64            # DC only: nnz 0
                else:
                    coeffs[m, 16 * i:16 * i + 16] = rng.integers(-64, 65, 16) * (rng.random(16) < 0.4) * 4
                    coeffs[m, 16 * i] = rng.integers(-600, 601)
                    nnzc[m, scan8(i + 4)] = 16
    if bits == 8:
        return rec, coeffs, nnzc
    return rec, coeffs.astype(np.int32) * (1 << (bits - 8)), nnzc
