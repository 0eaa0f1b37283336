"""Edge-case work for the H.264 batch calls and the layout they run in: the 8-bit ones (ff_h264_mc / idct_add_mb / weight /
deblock_*_cuda; tests/test_gpu_h264_edges.py, tests/test_h264_edges_cpu.py) and the 9 / 10-bit and 4:2:2 ones of h264_hbd_batch.cu
(tests/test_gpu_h264_hbd_edges.py, tests/test_h264_hbd_edges_cpu.py), which take the same generators at their sample size: `bits`
9 / 10 gives uint16 planes and int32 coefficients, and every offset, pad and shift stays in bytes.  TEST INFRASTRUCTURE.

The generators of libav_b200/synth.py stay as they are (bench.py and the older tests depend on their exact output); these reach what they
never produce: every partition shape with vectors up to the level limits, int16 wrap-around in both transform passes, the three dispatch
rules of h264_idct_add16 / add16intra / idct8_add4, every corner of the weighted-prediction parameters, and the high-qp rows of the
deblocking tables.  Each generator asserts that the cases it exists for really occur.  `Layout` puts a picture into decoder layout:
line sizes wider than the picture and planes inside poisoned allocations, so reads and writes of the row padding show."""
import numpy as np

from libav_b200 import synth
import h264_util as hu

MV_X, MV_Y = (-2048, 2048), (-2048, 2047)          # level limits of the vectors, quarter-pels (H.264 Table A-1, MaxVmvR at level >= 3.1)


# ---------------------------------------------------------------------------------------------------------------------------------
# decoder layout
# ---------------------------------------------------------------------------------------------------------------------------------
POISON = 0xA7
GUARD = 3                                           # guard rows above and below every plane


class Layout:
    """Line sizes and plane positions of one picture, in bytes: luma linesize = width * sample size + pad, chroma uvlinesize = its width *
    sample size + cpad; every plane sits `shift` (luma) / `cshift` (chroma) bytes past an aligned allocation, below GUARD poisoned rows.
    uint16 planes are placed byte for byte like uint8 ones (a POISON sample reads 0xA7A7, beyond every bit depth)."""

    def __init__(self, name, pad, cpad, shift=0, cshift=0, ref_shift=0):
        self.name, self.pad, self.cpad, self.shift, self.cshift, self.ref_shift = name, pad, cpad, shift, cshift, ref_shift

    def __repr__(self):
        return self.name

    def linesizes(self, w, sb=1):
        return w * sb + self.pad, w // 2 * sb + self.cpad

    def place(self, plane, chroma=False, ref=False):
        """(allocation, view): `plane` copied into an allocation of POISON bytes; the view is the picture inside it (at an odd byte
        position or pitch a uint16 view is unaligned: such layouts exist to be refused)"""
        h, w = plane.shape
        sb = plane.itemsize
        ls = w * sb + (self.cpad if chroma else self.pad)
        shift = self.ref_shift if ref else (self.cshift if chroma else self.shift)
        buf = np.full(shift + (h + 2 * GUARD) * ls, POISON, np.uint8)
        view = np.ndarray((h, w), plane.dtype, buffer=buf, offset=shift + GUARD * ls, strides=(ls, sb))
        view[...] = plane
        return buf, view

    @staticmethod
    def origin(buf, view):
        """byte offset of the picture's first sample in its allocation"""
        return view.ctypes.data - buf.ctypes.data

    @staticmethod
    def check(buf, view, want, what=""):
        """the picture equals `want`, and not one byte of the allocation outside it changed"""
        assert np.array_equal(view, want), (what, np.argwhere(view != want)[:5].tolist())
        outside = np.ones(buf.shape, bool)
        off, ls, wb = Layout.origin(buf, view), view.strides[0], view.shape[1] * view.itemsize
        for r in range(view.shape[0]):
            outside[off + r * ls:off + r * ls + wb] = False
        bad = np.flatnonzero(outside & (buf != POISON))
        assert bad.size == 0, (what, "bytes outside the picture changed", bad[:8].tolist())


# natural triggers of the fallback kernels (the launchers' conditions are quoted in the GPU tests)
PAD4 = Layout("pad4", 12, 4)                          # line sizes wider than the picture, all multiples of 4: the default kernels
PAD2 = Layout("pad2", 6, 6)                           # linesize = 2 mod 4
SHIFT1 = Layout("shift1", 4, 4, 1, 1)                 # every destination plane at +1 byte
SHIFT2 = Layout("shift2", 4, 4, 2, 2)                 # +2 bytes: chroma stays even, luma loses its word alignment
ODD_UV = Layout("odd_uv", 4, 3)                       # luma aligned, odd uvlinesize
ODD_CB = Layout("odd_cb", 4, 4, 0, 1)                 # luma aligned, chroma planes at odd addresses
REF1 = Layout("ref1", 4, 4, 0, 0, 1)                  # destination aligned, reference planes at +1 byte
# 16-bit samples (h264_hbd_batch.cu): pads and shifts stay even; PAD2, SHIFT2 and TIGHT / PAD4 serve as they are
REF2 = Layout("ref2", 4, 4, 0, 0, 2)                  # reference planes at +2 bytes, off 4-byte alignment
CSHIFT2 = Layout("cshift2", 8, 2, 0, 2)               # chroma planes at +2 bytes, uvlinesize = 2 mod 4, luma aligned
HBD_LAYOUTS = (PAD4, PAD2, SHIFT2, CSHIFT2)
# what the 16-bit calls refuse: an odd plane address (SHIFT1, ODD_CB), an odd uvlinesize (ODD_UV) or an odd linesize (ODD_LS)
ODD_LS = Layout("odd_ls", 3, 4)


# ---------------------------------------------------------------------------------------------------------------------------------
# motion compensation
# ---------------------------------------------------------------------------------------------------------------------------------
SUB = {"8x8": [(0, 0, 8, 8)], "8x4": [(0, 0, 8, 4), (0, 4, 8, 4)], "4x8": [(0, 0, 4, 8), (4, 0, 4, 8)],
       "4x4": [(x, y, 4, 4) for y in (0, 4) for x in (0, 4)]}
MB_SHAPES = {"16x16": [(0, 0, 16, 16)], "16x8": [(0, 0, 16, 8), (0, 8, 16, 8)], "8x16": [(0, 0, 8, 16), (8, 0, 8, 16)]}


def _vector(rng, x, y, w, h, pw, ph, regime):
    """a vector for the partition at (x, y): 'near' (+-64), 'far' (anywhere in the level range), 'limit' (a corner of the range) or
    'outside' (the partition's whole 6-tap window lies beyond one side or corner of the picture)"""
    if regime == "near":
        mv = rng.integers(-64, 65, size=2)
    elif regime == "far":
        mv = np.array([rng.integers(MV_X[0], MV_X[1] + 1), rng.integers(MV_Y[0], MV_Y[1] + 1)])
    elif regime == "limit":
        mv = np.array([MV_X[int(rng.integers(0, 2))], MV_Y[int(rng.integers(0, 2))]])
    else:
        while True:
            sx, sy = (int(v) for v in rng.integers(-1, 2, size=2))
            if sx or sy:
                break
        tx = -(w + 3) - int(rng.integers(0, 40)) if sx < 0 else pw + 3 + int(rng.integers(0, 40)) if sx > 0 else int(rng.integers(0, pw - w))
        ty = -(h + 3) - int(rng.integers(0, 40)) if sy < 0 else ph + 3 + int(rng.integers(0, 40)) if sy > 0 else int(rng.integers(0, ph - h))
        mv = np.array([4 * (tx - x) + int(rng.integers(0, 4)), 4 * (ty - y) + int(rng.integers(0, 4))])
    return int(np.clip(mv[0], *MV_X)), int(np.clip(mv[1], *MV_Y))


def mc_records(mb_w, mb_h, seed, nrefs=2, band=34):
    """Records covering every macroblock once with `put`, plus `avg` second directions on some partitions.  Every partition shape,
    8x4 and 4x8 as 8x8 sub-partitions (so 4x2 and 2x4 chroma blocks), all 16 quarter-sample positions, vectors up to the level
    limits and partitions wholly outside the picture on every side and corner.  The first `band` macroblocks are 16x16 partitions
    outside the picture and carry no `avg`: the first warp of 32 records holds 512 edge blocks, so its deferred-edge queue drains 16
    times."""
    rng = np.random.default_rng(seed)
    pw, ph = 16 * mb_w, 16 * mb_h
    out = []
    for m in range(mb_w * mb_h):
        mbx, mby = m % mb_w, m // mb_w
        if m < band:
            parts = MB_SHAPES["16x16"]
        else:
            kind = list(MB_SHAPES) + ["8x8"]
            k = kind[int(rng.integers(0, 4))]
            parts = MB_SHAPES[k] if k != "8x8" else \
                [(8 * (q & 1) + sx, 8 * (q >> 1) + sy, sw, sh) for q in range(4) for (sx, sy, sw, sh) in SUB[list(SUB)[int(rng.integers(0, 4))]]]
        for (px, py, w, h) in parts:
            x, y = 16 * mbx + px, 16 * mby + py
            regimes = ["outside"] if m < band else ["near", "near", "far", "outside", "limit"]
            for avg in (0, 1):
                if avg and (m < band or rng.random() >= 0.35):
                    break
                mvx, mvy = _vector(rng, x, y, w, h, pw, ph, regimes[int(rng.integers(0, len(regimes)))])
                out.append((x, y, mvx, mvy, w, h, avg, int(rng.integers(0, nrefs))))
    rec = np.zeros(len(out), synth.MC_DT)
    for k, name in enumerate(("x", "y", "mvx", "mvy", "w", "h", "avg", "ref")):
        rec[name] = [o[k] for o in out]
    shapes = {(int(r["w"]), int(r["h"])) for r in rec}
    assert shapes == {(16, 16), (16, 8), (8, 16), (8, 8), (8, 4), (4, 8), (4, 4)}, shapes
    pos = {(int(r["mvx"] + 4 * r["x"]) & 3) + 4 * (int(r["mvy"] + 4 * r["y"]) & 3) for r in rec}
    assert pos == set(range(16)), sorted(pos)
    assert rec["mvx"].min() == MV_X[0] and rec["mvx"].max() == MV_X[1] and rec["mvy"].min() == MV_Y[0] and rec["mvy"].max() == MV_Y[1]
    if band >= 32:
        assert all_edge_warps(rec, pw, ph) >= 1
    return rec


def mc_block_inside(pw, ph, mx, my):
    """h264_mc_block.cuh mc_block_inside() for a single picture with aligned planes: the block's patches are fetched as words"""
    sx, sy, cx, cy = (mx >> 2) - 2, (my >> 2) - 2, mx >> 3, my >> 3
    return sx >= 0 and (sx & ~3) + 12 <= pw and sy >= 0 and sy + 9 <= ph and cx >= 0 and (cx & ~3) + 8 <= (pw >> 1) and cy >= 0 and cy + 3 <= (ph >> 1)


def all_edge_warps(rec, pw, ph):
    """how many groups of 32 consecutive records (a warp of h264_mc_kernel_v2) hold `put` blocks that are all edge blocks"""
    n = 0
    for r0 in range(0, rec.shape[0] - 31, 32):
        blocks = [(int(r["mvx"]) + 4 * (int(r["x"]) + 4 * bx), int(r["mvy"]) + 4 * (int(r["y"]) + 4 * by))
                  for r in rec[r0:r0 + 32] if not r["avg"] for by in range(int(r["h"]) // 4) for bx in range(int(r["w"]) // 4)]
        n += len(blocks) > 32 and not any(mc_block_inside(pw, ph, mx, my) for mx, my in blocks)
    return n


def mc_pad(rec, pw, ph):
    """the padding oracle_mc needs around reference planes of pw x ph for these records: the farthest 6-tap / bilinear window"""
    mx = rec["mvx"].astype(np.int64) + 4 * rec["x"].astype(np.int64)
    my = rec["mvy"].astype(np.int64) + 4 * rec["y"].astype(np.int64)
    w, h = rec["w"].astype(np.int64), rec["h"].astype(np.int64)
    need = [-((mx >> 2) - 2).min(), ((mx >> 2) + w + 3 - pw).max(), -((my >> 2) - 2).min(), ((my >> 2) + h + 3 - ph).max(),
            -(mx >> 3).min(), ((mx >> 3) + w // 2 + 1 - pw // 2).max(), -(my >> 3).min(), ((my >> 3) + h // 2 + 1 - ph // 2).max()]
    return int(max(need + [1]))


def oracle_mc(o, rec, refs, dst, pw=None, ph=None):
    """the reference's qpel / chroma functions over `rec` in put-then-avg order (the batch call promises any record order), with the
    reference planes cropped to pw x ph and edge-replicated as far as the farthest vector reaches; returns the destination planes"""
    y = dst[0]
    pw, ph = pw or y.shape[1], ph or y.shape[0]
    pad = mc_pad(rec, pw, ph)
    if np.abs(rec["mvx"]).max() >= 1024:
        assert pad > 256, pad                         # the padding grew with the vectors
    crop = [(r[0][:ph, :pw], r[1][:ph >> 1, :pw >> 1], r[2][:ph >> 1, :pw >> 1]) for r in refs]
    order = np.concatenate([rec[rec["avg"] == 0], rec[rec["avg"] != 0]])
    want = [np.ascontiguousarray(p).copy() for p in dst]
    hu.oracle_mc(o, order, crop, *want, pad=pad)
    return want


# ---------------------------------------------------------------------------------------------------------------------------------
# residual
# ---------------------------------------------------------------------------------------------------------------------------------
DC_EDGE = list(range(32735, 32768)) + [-32768]
KINDS = ("none", "dense", "dc_wrap", "single_ac", "dc_and_ac", "dc_nnz0", "dc_nnz1")     # dc_wrap: DC at an end of coeff_range(bits)
CHROMA_422_LOWER = [20, 21, 22, 23, 36, 37, 38, 39]      # h264_idct_add8_422: rows 8..15 of each plane, nnz at scan8[i + 4]


def coeff_range(bits):
    """(lo, hi, DC values at the end of the range): 8 bit = the whole int16 range, where block[0] + 32 wraps in the reference's int16
    arithmetic; 9 / 10 bit = the legal range -2^(7 + bits) .. 2^(7 + bits) - 1 of int32 coefficients (no signed overflow in the
    reference's int arithmetic anywhere inside it)"""
    if bits == 8:
        return -32768, 32767, DC_EDGE
    lim = 1 << (7 + bits)
    return -lim, lim - 1, [lim - 1, lim - 2, lim - 33, -lim, -lim + 1]


def route(mode, chroma, nnz, dc):
    """what h264_idct_add16 (mode 0) / add16intra (1) / idct8_add4 (2) / idct_add8 / idct_add8_422 (chroma) do with a block: full, dc
    or skip (h264idct_template.c:174-236)"""
    if chroma or mode == 1:
        return "full" if nnz else "dc" if dc else "skip"
    return "skip" if not nnz else "dc" if nnz == 1 and dc else "full"


def _first_pass_wraps(b):
    """does the first (vertical) pass of ff_h264_idct_add on the 4x4 block b store a value outside int16?"""
    c = [int(v) for v in b]
    c[0] = (c[0] + 32 + 32768) % 65536 - 32768                           # block[0] += 32, stored as int16
    for i in range(4):
        z0, z1 = c[i] + c[i + 8], c[i] - c[i + 8]
        z2, z3 = (c[i + 4] >> 1) - c[i + 12], c[i + 4] + (c[i + 12] >> 1)
        if max(abs(z0 + z3), abs(z1 + z2), abs(z1 - z2), abs(z0 - z3)) > 32767:
            return True
    return False


def residual_records(mb_w, mb_h, seed, modes=(0, 1, 2, 3), bits=8, c422=0):
    """Records (tight layout: linesize 16 * mb_w samples, offsets in bytes), coefficient arena (n, 768; int16 at 8 bit, int32 above)
    and nnzc (n, 120).  Macroblocks cycle through `modes` with chroma on and off; every block of the arena is filled whatever the
    macroblock's mode, so blocks the dispatchers skip must come back untouched.  Block kinds: dense over the whole coefficient range
    (at random scales), DC at the ends of the range with dense AC, nnz 1 with DC 0 and one AC coefficient, nnz 1 with DC and AC both
    nonzero, nnz 0 with a DC, and the plain DC-only block.  c422: the lower four chroma blocks of each plane as well."""
    rng = np.random.default_rng(seed)
    lo, hi, dc_edge = coeff_range(bits)
    sb = 1 if bits == 8 else 2
    n, W = mb_w * mb_h, 16 * mb_w * sb
    rec = np.zeros(n, synth.RESIDUAL_DT)
    m = np.arange(n)
    rec["luma_off"] = (m // mb_w) * 16 * W + (m % mb_w) * 16 * sb
    rec["chroma_off"] = (m // mb_w) * (16 if c422 else 8) * (W // 2) + (m % mb_w) * 8 * sb
    rec["luma_mode"] = np.array(modes, np.uint8)[m % len(modes)]
    rec["chroma"] = (m // len(modes)) % 2
    coeffs = np.zeros((n, 768), np.int16 if bits == 8 else np.int32)
    nnzc = np.zeros((n, 120), np.uint8)
    seen = {}
    wrap_dc = 0
    for mb in range(n):
        mode = int(rec["luma_mode"][mb])
        for i in list(range(16)) + [16, 17, 18, 19, 32, 33, 34, 35] + (CHROMA_422_LOWER if c422 else []):
            is_chroma = i >= 16
            size = 64 if mode == 2 and not is_chroma else 16
            if size == 64 and i & 3:
                continue                                                       # covered by the 8x8 block i & ~3
            kind = KINDS[int(rng.integers(0, len(KINDS)))]
            b = np.zeros(size, np.int64)
            nnz = 0
            if kind in ("dense", "dc_wrap"):
                scale = 1 << int(rng.integers(4, 8 + bits))
                b = rng.integers(-scale, scale, size=size)
                b[rng.random(size) < 0.1] = rng.choice([lo, hi])
                if kind == "dc_wrap":
                    b[0] = dc_edge[int(rng.integers(0, len(dc_edge)))]
                nnz = int(rng.integers(2, 17))
            elif kind == "single_ac":
                b[int(rng.integers(1, size))] = rng.integers(lo, hi + 1) or 1
                nnz = 1
            elif kind == "dc_and_ac":
                b[0] = rng.choice([int(rng.integers(lo, hi + 1)) or 5, dc_edge[int(rng.integers(0, len(dc_edge)))]])
                b[1 + rng.choice(size - 1, int(rng.integers(1, 4)), replace=False)] = rng.integers(1, 3000)
                nnz = 1
            elif kind in ("dc_nnz0", "dc_nnz1"):
                b[0] = rng.choice([int(rng.integers(lo, hi + 1)) or 7, dc_edge[int(rng.integers(0, len(dc_edge)))]])
                nnz = 0 if kind == "dc_nnz0" else 1
            coeffs[mb, 16 * i:16 * i + size] = b.astype(coeffs.dtype)
            nnzc[mb, synth.scan8(i + 4 if i in CHROMA_422_LOWER else i)] = nnz
            visited = is_chroma and rec["chroma"][mb] or not is_chroma and mode < 3
            if not visited:
                continue
            r = route(mode, is_chroma, nnz, int(b[0]))
            key = ("chroma422_lower" if i in CHROMA_422_LOWER else "chroma" if is_chroma else "luma%d" % mode, kind, r)
            seen[key] = seen.get(key, 0) + 1
            if r == "full" and bits == 8 and b[0] + 32 > 32767:
                wrap_dc += 1
                if size == 16 and _first_pass_wraps(b):
                    seen["first_pass_wrap"] = seen.get("first_pass_wrap", 0) + 1
    # the cases this generator exists for
    combos = {(int(a), int(c)) for a, c in zip(rec["luma_mode"], rec["chroma"])}
    assert combos == {(md, c) for md in modes for c in (0, 1)}, combos
    if bits == 8:
        assert wrap_dc > 0 and seen.get("first_pass_wrap", 0) > 0
    else:
        assert coeffs.min() == lo and coeffs.max() == hi, (coeffs.min(), coeffs.max())
    assert seen.get(("chroma", "dc_wrap", "full"), 0) > 0 and seen.get(("chroma", "dc_nnz0", "dc"), 0) > 0
    if c422:
        for k in (("dc_wrap", "full"), ("dc_nnz0", "dc"), ("single_ac", "full"), ("none", "skip")):
            assert seen.get(("chroma422_lower",) + k, 0) > 0, k
    for md in modes:
        if md == 0 or md == 2:
            assert seen.get(("luma%d" % md, "single_ac", "full"), 0) > 0           # nnz 1, DC 0: the full transform
            assert seen.get(("luma%d" % md, "dc_and_ac", "dc"), 0) > 0             # nnz 1, DC and AC: DC only, the AC stays
            assert seen.get(("luma%d" % md, "dc_wrap", "full"), 0) > 0
            assert seen.get(("luma%d" % md, "dc_nnz0", "skip"), 0) > 0             # nnz 0 with a DC: skipped
        if md == 1:
            assert seen.get(("luma1", "dc_nnz0", "dc"), 0) > 0 and seen.get(("luma1", "dc_wrap", "full"), 0) > 0
    return rec, coeffs, nnzc


def relayout_residual(rec, W, ls, uvls):
    """records with tight offsets (linesize W bytes, chroma W / 2) moved to line sizes ls / uvls"""
    out = rec.copy()
    out["luma_off"] = (rec["luma_off"] // W) * ls + rec["luma_off"] % W
    out["chroma_off"] = (rec["chroma_off"] // (W // 2)) * uvls + rec["chroma_off"] % (W // 2)
    return out


DC_DT = np.dtype([("luma_qmul", "<u4"), ("chroma_qmul", "<u4", (2,))])          # FFH264DCRecord
DC_QMUL = (0, 1, 16, 255, 4096, 1 << 16, 1 << 20)


def dc_records(n, bits, c422, seed):
    """FFH264DCRecord per macroblock at 9 / 10 bit, the luma DC blocks (n, 16) and a coefficient arena (n, 768) int32 whose chroma DC
    positions hold the chroma DC levels: qmul over DC_QMUL (0: the plane is skipped), levels at the ends of the legal range
    +-2^(7 + bits), scaled down where needed so that the reference's int arithmetic -- (sum of up to 16 levels) * qmul + 128 -- stays
    inside int32; every other coefficient of the arena is noise the call must leave alone."""
    rng = np.random.default_rng(seed)
    lo, hi, _ = coeff_range(bits)
    rec = np.zeros(n, DC_DT)
    rec["luma_qmul"] = rng.choice(DC_QMUL, n)
    rec["chroma_qmul"] = rng.choice(DC_QMUL, (n, 2))
    coeffs = rng.integers(lo, hi + 1, size=(n, 768)).astype(np.int32)
    luma_dc = np.zeros((n, 16), np.int32)
    ndc = 8 if c422 else 4

    def levels(qmul, k):
        bound = ((1 << 31) - 256) // (16 * max(int(qmul), 1))
        neg, pos = -min(-lo, bound), min(hi, bound)
        return rng.choice([neg, neg + 1, pos, pos - 1, 0], k) if rng.random() < 0.5 else rng.integers(neg, pos + 1, k)
    near_limit = 0
    for m in range(n):
        luma_dc[m] = levels(rec["luma_qmul"][m], 16)
        near_limit += int(np.abs(luma_dc[m]).sum()) * int(rec["luma_qmul"][m]) >= 1 << 30
        for p in range(2):
            coeffs[m, 256 * (p + 1):256 * (p + 1) + 16 * ndc:16] = levels(rec["chroma_qmul"][m, p], ndc)
    assert luma_dc.min() == lo and luma_dc.max() == hi and near_limit > 0
    assert {0, 1 << 20} <= set(rec["luma_qmul"].tolist()) and {0, 1 << 20} <= set(rec["chroma_qmul"].ravel().tolist())
    return rec, coeffs, luma_dc


# ---------------------------------------------------------------------------------------------------------------------------------
# weighted prediction
# ---------------------------------------------------------------------------------------------------------------------------------
WEIGHTS, OFFSETS = (-128, -1, 0, 1, 127), (-128, 0, 127)
HEIGHTS = {16: (16, 8), 8: (16, 8, 4), 4: (8, 4, 2), 2: (4, 2)}         # the heights mc_part_weighted() passes per width


def weight_records(bi, seed, cols=32, bits=8):
    """Every corner: log2_denom 0..7 x weight {-128, -1, 0, 1, 127} x offset {-128, 0, 127} (bi: x the same weights for the second
    prediction, cycled) x width 16 / 8 / 4 / 2 x content 0 / 2^bits - 1 / noise.  One record per 16 x 16 slot of the plane (tight,
    linesize 16 * cols samples; offsets in bytes).  Returns (records, destination plane, second-prediction plane)."""
    rng = np.random.default_rng(seed)
    combos = [(ld, w, o, wd, c) for ld in range(8) for w in WEIGHTS for o in OFFSETS for wd in (16, 8, 4, 2) for c in range(3)]
    rows = -(-len(combos) // cols)
    W, top, sb = 16 * cols, (1 << bits) - 1, 1 if bits == 8 else 2
    dt = np.uint8 if bits == 8 else np.uint16
    plane = rng.integers(0, top + 1, size=(16 * rows, W), dtype=dt)
    src = rng.integers(0, top + 1, size=(16 * rows, W), dtype=dt)
    rec = np.zeros(len(combos), synth.WEIGHT_DT)
    for k, (ld, w, o, wd, c) in enumerate(combos):
        y0, x0 = 16 * (k // cols), 16 * (k % cols)
        if c < 2:
            plane[y0:y0 + 16, x0:x0 + 16] = top * c
            src[y0:y0 + 16, x0:x0 + 16] = top * (c if k % 2 else 1 - c)
        rec[k] = ((y0 * W + x0) * sb, wd, HEIGHTS[wd][k % len(HEIGHTS[wd])], ld, 0, w, WEIGHTS[(k // 7) % 5] if bi else 0, o, 0)
    return rec, plane, src


def relayout_offsets(off, W, ls):
    return (off // W) * ls + off % W


# ---------------------------------------------------------------------------------------------------------------------------------
# deblocking
# ---------------------------------------------------------------------------------------------------------------------------------
# H.264 Tables 8-16 and 8-17: alpha', beta' by indexA / indexB, tC0' by indexA and bS 1..3
ALPHA = np.array([0] * 16 + [4, 4, 5, 6, 7, 8, 9, 10, 12, 13, 15, 17, 20, 22, 25, 28, 32, 36, 40, 45, 50, 56, 63, 71, 80, 90, 101, 113,
                             127, 144, 162, 182, 203, 226, 255, 255])
BETA = np.array([0] * 16 + [2, 2, 2, 3, 3, 3, 3, 4, 4, 4, 6, 6, 7, 7, 8, 8, 9, 9, 10, 10, 11, 11, 12, 12, 13, 13, 14, 14, 15, 15, 16, 16,
                            17, 17, 18, 18])
TC0 = np.array([[0, 0, 0]] * 17 + [[0, 0, 1]] * 4 + [[0, 1, 1]] * 2 + [[1, 1, 1]] * 4 + [[1, 1, 2]] * 4 +
               [[1, 2, 3], [1, 2, 3], [2, 2, 3], [2, 2, 4], [2, 3, 4], [2, 3, 4], [3, 3, 5], [3, 4, 6], [3, 4, 6], [4, 5, 7], [4, 5, 8],
                [4, 6, 9], [5, 7, 10], [6, 8, 11], [6, 8, 13], [7, 10, 14], [8, 11, 16], [9, 12, 18], [10, 13, 20], [11, 15, 23],
                [13, 17, 25]])
assert ALPHA.shape == (52,) and BETA.shape == (52,) and TC0.shape == (52, 3)


def deblock_records(mb_w, mb_h, seed, with_qp=False):
    """Per edge: qp over the whole 0..51 range, slice index offsets -12..12 (FilterOffsetA / B), alpha / beta / tc0 from the
    standard's tables (chroma through the chroma qp table), bS 0..3 per group of four lines, bS 4 on some macroblock edges.
    Picture-boundary edges carry alpha = 0 like synth.h264_deblock_work.  with_qp: also the qp of every edge, (n, 2, 4).  The table
    corners are asserted from 32 macroblocks on (a smaller picture has too few edges to reach them all)."""
    rng = np.random.default_rng(seed)
    n = mb_w * mb_h
    rec = np.zeros(n, synth.DEBLOCK_DT)
    qps = np.zeros((n, 2, 4), np.int64)
    for m in range(n):
        for d in (0, 1):
            for e in range(4):
                qp = int(rng.integers(0, 52)) if rng.random() < 0.5 else int(rng.integers(36, 52))
                qps[m, d, e] = qp
                oa, ob = (int(v) for v in rng.integers(-12, 13, size=2))
                ia, ib = np.clip(qp + oa, 0, 51), np.clip(qp + ob, 0, 51)
                rec["alpha"][m, d, e], rec["beta"][m, d, e] = ALPHA[ia], BETA[ib]
                intra = e == 0 and rng.random() < 0.3
                rec["intra"][m, d] |= intra << e
                bs = rng.integers(0, 4, size=4)
                rec["tc0"][m, d, e] = np.where(bs > 0, TC0[ia][np.maximum(bs - 1, 0)], -1)
                if not (e & 1):
                    for p in range(2):
                        cq = int(synth.H264_CHROMA_QP[qp])
                        ca, cb = np.clip(cq + oa, 0, 51), np.clip(cq + ob, 0, 51)
                        rec["calpha"][m, p, d, e >> 1], rec["cbeta"][m, p, d, e >> 1] = ALPHA[ca], BETA[cb]
                        rec["cintra"][m, p, d] |= intra << (e >> 1)
                        rec["ctc0"][m, p, d, e >> 1] = np.where(bs > 0, TC0[ca][np.maximum(bs - 1, 0)] + 1, 0)
        if m % mb_w == 0:
            rec["alpha"][m, 0, 0] = 0; rec["calpha"][m, :, 0, 0] = 0
        if m < mb_w:
            rec["alpha"][m, 1, 0] = 0; rec["calpha"][m, :, 1, 0] = 0
    if n >= 32:
        assert rec["alpha"].max() == 255 and rec["tc0"].max() == 25 and rec["ctc0"].max() >= 20 and rec["beta"].max() == 18
        strong = (rec["intra"][:, :, None] & 1).astype(bool) & (rec["alpha"][:, :, :1] >= 200)
        assert strong.any()                                              # bS 4 with (alpha >> 2) + 2 >= 52
    return (rec, qps) if with_qp else rec


def deblock422_records(mb_w, mb_h, seed):
    """4:2:2 pictures: (104-byte records, the matching 52-byte FFH264DeblockChroma422 records, qp per edge).  The four horizontal
    chroma edges of a macroblock (rows 0, 4, 8, 12) take the qp and the intra flag of the luma edge of the same index, alpha / beta /
    tc0 + 1 from the tables through the chroma qp table with their own offsets and bS; the picture's top edge carries alpha = 0."""
    rec, qps = deblock_records(mb_w, mb_h, seed, with_qp=True)
    rng = np.random.default_rng(seed + 1000)
    n = mb_w * mb_h
    ext = np.zeros(n, CHROMA422_DT)
    for m in range(n):
        for p in range(2):
            for e in range(4):
                cq = int(synth.H264_CHROMA_QP[qps[m, 1, e]])
                oa, ob = (int(v) for v in rng.integers(-12, 13, size=2))
                ca, cb = np.clip(cq + oa, 0, 51), np.clip(cq + ob, 0, 51)
                ext["alpha"][m, p, e], ext["beta"][m, p, e] = ALPHA[ca], BETA[cb]
                bs = rng.integers(0, 4, size=4)
                ext["tc0"][m, p, e] = np.where(bs > 0, TC0[ca][np.maximum(bs - 1, 0)] + 1, 0)
            ext["intra"][m, p] = rec["intra"][m, 1] & 1
        if m < mb_w:
            ext["alpha"][m, :, 0] = 0
    if n >= 32:
        assert ext["alpha"].max() >= 200 and ext["tc0"].max() >= 20 and (ext["intra"] & 1).any()
    return rec, ext, qps


CHROMA422_DT = np.dtype([("alpha", "u1", (2, 4)), ("beta", "u1", (2, 4)), ("tc0", "i1", (2, 4, 4)), ("intra", "u1", (2,)), ("pad", "u1", (2,))])
assert CHROMA422_DT.itemsize == 52                       # FFH264DeblockChroma422


def blocky(shape, seed, bits=8):
    """4x4 blocks of flat content (+-1 of noise, both scaled by 2^(bits - 8)) whose steps range up to 2^bits - 1: large alpha and tc
    let the filters act on big steps"""
    rng = np.random.default_rng(seed)
    h, w = shape
    sc = 1 << (bits - 8)
    scale = rng.choice([8, 32, 96, 255], size=(h // 16 + 1, w // 16 + 1))
    base = 128 + (rng.random((h // 4 + 1, w // 4 + 1)) - 0.5) * np.kron(scale, np.ones((4, 4)))[:h // 4 + 1, :w // 4 + 1]
    up = np.kron(base, np.ones((4, 4)))[:h, :w]
    v = np.clip(up * sc + rng.integers(-1, 2, size=shape) * sc, 0, (1 << bits) - 1)
    return v.astype(np.uint8 if bits == 8 else np.uint16)


def high_qp_edges_changed(qps, mb_w, mb_h, before, after, qp_min=40):
    """how many luma samples next to an edge whose record comes from qp >= qp_min the filters changed: the samples p0 / q0 on both
    sides of every vertical and horizontal edge"""
    n = 0
    for m in np.argwhere((qps >= qp_min).any(axis=(1, 2))).ravel():
        y0, x0 = 16 * (m // mb_w), 16 * (m % mb_w)
        for d, e in np.argwhere(qps[m] >= qp_min):
            if d == 0 and x0 + 4 * e > 0:
                sl = np.s_[y0:y0 + 16, x0 + 4 * e - 1:x0 + 4 * e + 1]
            elif d == 1 and y0 + 4 * e > 0:
                sl = np.s_[y0 + 4 * e - 1:y0 + 4 * e + 1, x0:x0 + 16]
            else:
                continue
            n += int((before[sl] != after[sl]).sum())
    return n
