"""Edge-case work for the batched H.264 intra reconstruction (ff_h264_intra_mb_batch_cuda, and the _hbd / _422 calls that read the same
FFH264IntraMB records), shaped like the decoder.  Shared by tests/test_gpu_h264_intra_edges.py and tests/test_h264_intra_edges_cpu.py.
TEST INFRASTRUCTURE.

synth.h264_intra_work stays as it is (bench.py and the older tests depend on its exact output).  Its pictures are one slice without
constrained_intra_pred, so every neighbour inside the picture is available, and its coefficients are small.  The pictures here have
raster-scan slices that start anywhere (column 0, mid-row, column mb_w - 1, one-macroblock slices) and constrained_intra_pred on or off, so
top, top-left and top-right can be unavailable in mid-picture, where the kernel must follow the masks and not the geometry:
  masks  fill_decode_caches(), non-MBAFF branch (libavcodec/h264_mvpred.h:466-508), from the neighbours' availability
  modes  drawn as coded, then passed through ff_h264_check_intra4x4_pred_mode / ff_h264_check_intra_pred_mode (h264_parse.c:103-189):
         the substitutions are applied, a refused mode is drawn again
  arena  every block of every macroblock carries one of the residual kinds of h264_edge_cases.py (int16 wrap-around, the dispatch rules),
         inter macroblocks and the chroma of chroma_residual = 0 included: those must come back untouched, like elements 576..767
  samples  per macroblock noise, flat 0, flat max or a 0 / max checkerboard, so prediction and the residual clip at both ends
`intra_case` returns what it covered; `assert_coverage` holds the union of the matrix below to every case it exists for."""
import collections
import functools
from itertools import repeat

import numpy as np

from libav_b200 import synth
import h264_edge_cases as ec
from h264_util import scan8

SIZES = [(1, 1), (1, 68), (2, 3), (3, 2), (11, 7), (120, 68)]
VARIANTS = [(False, False), (True, False), (False, True), (True, True)]            # (slices, constrained_intra_pred)
ARENA_POISON = 0x5A5A                                                               # arena elements no block owns (int16; int32: 0x5A5A5A5A)

# ff_h264_check_intra4x4_pred_mode's top[] / left[] and ff_h264_check_intra_pred_mode's (h264_parse.c): < 0 refused, > 0 substituted
TOP4 = (-1, 0, 9, -1, -1, -1, -1, -1, 0, 0, 0, 0)
LEFT4 = (0, -1, 10, 0, -1, -1, -1, 0, -1, 11, 0, 0)
TOP16, LEFT16 = (4, 1, -1, -1), (5, -1, 2, -1, 6)
DC_128_PRED, PLANE_PRED8x8, DC_128_PRED8x8 = 11, 3, 6


def masks(top, left, topleft, topright):
    """(topleft, top, left, topright)_samples_available of an intra macroblock whose neighbours are available or not"""
    tl, t, lm, tr = 0xFFFF, 0xFFFF, 0xFFFF, 0xEEEA
    if not top:
        tl, t, tr = 0xB3FF, 0x33FF, 0x26EA
    if not left:
        tl &= 0xDF5F
        lm &= 0x5F5F
    if not topleft:
        tl &= 0x7FFF
    if not topright:
        tr &= 0xFBFF
    return tl, t, lm, tr


def tl_tr8(tl_mask, tr_mask, k):
    """has_topleft / has_topright of 8x8 block k as hl_decode_mb_predict_luma passes them to pred8x8l"""
    return int(bool((tl_mask << 4 * k) & 0x8000)), int(bool((tr_mask << 4 * k) & 0x4000))


# the (has_topleft, has_topright) pairs the masks can give each 8x8 block: all four for blocks 0 and 1, the lower blocks have fewer
TLTR8 = [{tl_tr8(m[0], m[3], k) for m in (masks(*((a >> b) & 1 for b in range(4))) for a in range(16))} for k in range(4)]


def check4(mode, top, left):
    """ff_h264_check_intra4x4_pred_mode on one entry: the mode after substitution, None if refused"""
    for ok, tab in ((top, TOP4), (left, LEFT4)):
        if not ok:
            s = tab[mode]
            if s < 0:
                return None
            mode = s or mode
    return mode


def check16(mode, top, left):
    """ff_h264_check_intra_pred_mode for 16x16 and (non-MBAFF) chroma"""
    if not top:
        mode = TOP16[mode]
        if mode < 0:
            return None
    if not left:
        mode = LEFT16[mode]
    return mode if mode >= 0 else None


@functools.lru_cache(maxsize=None)
def accepted(check, n_coded, top, left):
    return [check(m, top, left) for m in range(n_coded) if check(m, top, left) is not None]


def draw(rng, check, n_coded, top, left):
    """a coded mode 0..n_coded - 1 the check accepts (drawing again on refusal is drawing among the accepted ones), after substitution"""
    ok = accepted(check, n_coded, bool(top), bool(left))
    return ok[int(rng.integers(0, len(ok)))]


def first_pass_wraps8(b):
    """does the first (column) pass of ff_h264_idct8_add on the 8x8 block b store a value outside int16?"""
    c = np.array(b, np.int64).reshape(8, 8).copy()
    c[0, 0] = (c[0, 0] + 32 + 32768) % 65536 - 32768                   # block[0] += 32, stored as int16
    s = [c[k] for k in range(8)]                                       # row k of every column at once
    a0, a2, a4, a6 = s[0] + s[4], s[0] - s[4], (s[2] >> 1) - s[6], (s[6] >> 1) + s[2]
    b0, b2, b4, b6 = a0 + a6, a2 + a4, a2 - a4, a0 - a6
    a1 = -s[3] + s[5] - s[7] - (s[7] >> 1)
    a3 = s[1] + s[7] - s[3] - (s[3] >> 1)
    a5 = -s[1] + s[7] + s[5] + (s[5] >> 1)
    a7 = s[3] + s[5] + s[1] + (s[1] >> 1)
    b1, b3, b5, b7 = (a7 >> 2) + a1, a3 + (a5 >> 2), (a3 >> 2) - a5, a7 - (a1 >> 2)
    out = np.stack([b0 + b7, b2 + b5, b4 + b3, b6 + b1, b6 - b1, b4 - b3, b2 - b5, b0 - b7])
    return bool(np.abs(out).max() > 32767)


def blocks(rng, n, size):
    """n coefficient blocks of `size` (16, or 64 for 8x8), each of one of ec.KINDS: nothing; dense over the full int16 range at a random
    scale; dense with DC at 32735..32767 / -32768; nnz 1 with DC 0 and one AC; nnz 1 with DC and AC; DC with nnz 0; DC with nnz 1.
    Returns (kind names, values int64 (n, size), nnz)"""
    name = np.array(ec.KINDS)[rng.integers(0, len(ec.KINDS), n)]
    scale = (1 << rng.integers(4, 16, n))[:, None]
    dense = rng.integers(-scale, scale, (n, size))
    ext = rng.random((n, size)) < 0.1
    dense[ext] = rng.choice([-32768, 32767], int(ext.sum()))
    edge = np.array(ec.DC_EDGE)[rng.integers(0, len(ec.DC_EDGE), n)]
    dc = np.where(rng.random(n) < 0.5, rng.integers(-32768, 32768, n), edge)
    dc[dc == 0] = 7
    b = np.zeros((n, size), np.int64)
    nnz = np.zeros(n, np.int64)
    d = np.isin(name, ("dense", "dc_wrap"))
    b[d] = dense[d]
    nnz[d] = rng.integers(2, 17, n)[d]
    w = name == "dc_wrap"
    b[w, 0] = edge[w]
    s = np.flatnonzero(name == "single_ac")
    val = rng.integers(-32768, 32768, n)
    val[val == 0] = 1
    b[s, rng.integers(1, size, n)[s]] = val[s]
    nnz[s] = 1
    a = name == "dc_and_ac"
    ac = (rng.random((n, size)) < 3.0 / size) * rng.integers(1, 3000, (n, size))
    ac[np.arange(n), rng.integers(1, size, n)] = rng.integers(1, 3000, n)
    ac[:, 0] = dc
    b[a] = ac[a]
    nnz[a] = 1
    for k, c in (("dc_nnz0", 0), ("dc_nnz1", 1)):
        m = name == k
        b[m, 0] = dc[m]
        nnz[m] = c
    return name, b, nnz


def picture(mb_w, mb_h, rng, bits=8, c422=0):
    """luma, cb, cr: each macroblock's area noise, flat 0, flat max or a 0 / max checkerboard"""
    top = (1 << bits) - 1

    def plane(bh, bw):
        h, w = bh * mb_h, bw * mb_w
        yy, xx = np.mgrid[0:h, 0:w]
        pick = np.kron(rng.integers(0, 4, (mb_h, mb_w)), np.ones((bh, bw), np.int64))
        p = np.select([pick == 0, pick == 1, pick == 2], [rng.integers(0, top + 1, (h, w)), 0, top], ((yy + xx) & 1) * top)
        return p.astype(np.uint8 if bits == 8 else np.uint16)
    ch = 16 if c422 else 8
    return plane(16, 16), plane(ch, 8), plane(ch, 8)


def slice_map(mb_w, mb_h, rng, slices):
    """slice index of each macroblock: raster-scan slices starting at column 0, mid-row, at column mb_w - 1, one-macroblock slices and
    at random places"""
    n = mb_w * mb_h
    if not slices:
        return np.zeros(n, np.int64)
    mid = (mb_h // 2) * mb_w
    starts = np.zeros(n, bool)
    starts[[s for s in (mid, mid + mb_w // 2, mid + mb_w // 2 + 1, mid + mb_w - 1, n - 1) if 0 < s < n]] = True
    starts |= rng.random(n) < max(0.01, min(0.2, 6.0 / n))
    starts[0] = False
    return np.cumsum(starts)


def intra_case(mb_w, mb_h, seed, slices, constrained, bits=8, c422=0):
    """One picture: records, coefficient arena (n, 768) (int16 at 8 bit; at 9 / 10 bit the same kinds as int32 scaled by 32, up to
    +-2^20, where the reference's int arithmetic cannot overflow), nnzc (n, 120), planes, and a Counter of the cases it covered."""
    rng = np.random.default_rng(seed)
    n = mb_w * mb_h
    sl = slice_map(mb_w, mb_h, rng, slices)
    kind = rng.choice(4, n, p=[0.2, 0.3, 0.3, 0.2])
    if not kind.any():
        kind[0] = 1
    rec = np.zeros(n, synth.INTRA_DT)
    coeffs = np.zeros((n, 768), np.int64)
    nnzc = rng.integers(0, 256, (n, 120)).astype(np.uint8)      # entries no block reads hold anything
    seen = collections.Counter()

    def avail(m, nx, ny):
        q = ny * mb_w + nx
        return 0 <= nx < mb_w and ny >= 0 and sl[q] == sl[m] and not (constrained and kind[q] == 0)

    for m in range(n):
        x, y = m % mb_w, m // mb_w
        k = int(kind[m])
        t, l, tl, tr = avail(m, x, y - 1), avail(m, x - 1, y), avail(m, x - 1, y - 1), avail(m, x + 1, y - 1)
        tl_m, _, _, tr_m = masks(t, l, tl, tr)
        mid = x > 0 and y > 0
        r = rec[m]
        r["kind"] = k
        r["chroma_residual"] = rng.random() < 0.6
        r["mode4"] = rng.integers(0, 12, 16)                               # kind 2 reads entries 0, 4, 8, 12; kind 0 / 3 none
        if k == 0:                                                        # not intra: the rest of the record means nothing
            r["mode16"], r["chroma_mode"] = rng.integers(0, 7, 2)
            r["topleft"], r["topright"] = rng.integers(0, 1 << 16, 2)
        else:
            r["topleft"], r["topright"] = tl_m, tr_m
            r["chroma_mode"] = draw(rng, check16, 4, t, l)
            if k == 3:
                r["mode16"] = draw(rng, check16, 4, t, l)
            for big, what in ((int(r["chroma_mode"]), "chroma"), (int(r["mode16"]) if k == 3 else -1, "luma")):
                if big == PLANE_PRED8x8 and constrained and x > 0 and y > 0 and sl[m - mb_w - 1] == sl[m] and kind[m - mb_w - 1] == 0:
                    seen["plane_inter_topleft", what] += 1                 # PLANE still reads the corner sample
                if big == DC_128_PRED8x8 and mid:
                    seen["dc128_mid"] += 1
            if not t and y > 0:
                seen["top_unavailable_mid"] += 1
            if k in (1, 2):
                for i in range(0, 16, 1 if k == 1 else 4):
                    top_row, left_col = i in (0, 1, 4, 5), i in (0, 2, 8, 10)
                    md = draw(rng, check4, 9, t or not top_row, l or not left_col)
                    r["mode4"][i] = md
                    seen["mode%d" % (4 if k == 1 else 8), md] += 1
                    if md == DC_128_PRED and mid:
                        seen["dc128_mid"] += 1
                    trb = bool((tr_m << i) & (0x8000 if k == 1 else 0x4000))
                    if k == 1 and i == 5 and not trb and x + 1 < mb_w and y > 0 and md in (3, 7):
                        seen["tr_unavailable_4x4_block5"] += 1             # DIAG_DOWN_LEFT / VERT_LEFT repeat the last top sample
                    if k == 2:
                        seen["tltr", i // 4, tl_tr8(tl_m, tr_m, i // 4)] += 1
                        if i == 4 and not trb and x + 1 < mb_w:
                            seen["tr_unavailable_8x8_block1"] += 1
                        if i == 0 and mid and not tl_tr8(tl_m, tr_m, 0)[0]:
                            seen["tl_unavailable_8x8_block0"] += 1
    # coefficients: every block of every macroblock, whoever reads it.  Luma 4x4 blocks 0..15 and 8x8 blocks 0 / 4 / 8 / 12 both fill
    # elements 0..255; chroma blocks 16.. / 32.. (4:2:2: 8 per plane, the lower four counted at scan8[i + 4])
    l4, l8 = blocks(rng, 16 * n, 16), blocks(rng, 4 * n, 64)
    is8 = kind == 2
    coeffs[:, :256] = np.where(is8[:, None], l8[1].reshape(n, 256), l4[1].reshape(n, 256))
    for i in range(16):
        nnzc[~is8, scan8(i)] = l4[2].reshape(n, 16)[~is8, i]
    for q in range(4):                                          # the other three entries keep random counts, as CAVLC leaves them
        nnzc[is8, scan8(4 * q)] = l8[2].reshape(n, 4)[is8, q]
    chroma_blocks = [16 * p + k for p in (1, 2) for k in range(8 if c422 else 4)]
    cb_ = blocks(rng, len(chroma_blocks) * n, 16)
    for j, i in enumerate(chroma_blocks):
        coeffs[:, 16 * i:16 * i + 16] = cb_[1].reshape(n, -1, 16)[:, j]
        nnzc[:, scan8(i + 4 if i & 4 else i)] = cb_[2].reshape(n, -1)[:, j]
    owned = np.zeros(768, bool)
    owned[:256] = True
    for i in chroma_blocks:
        owned[16 * i:16 * i + 16] = True

    # what each block meets: its region's dispatch rule (h264_edge_cases.route), or nothing (inter macroblocks, chroma without residual)
    def tally(region, names, vals, nnz, read, add16):
        dc = vals[:, 0] != 0
        rt = np.where(nnz == 0, np.where(add16 & dc, "dc", "skip"), np.where((not add16) & (nnz == 1) & dc, "dc", "full"))
        seen.update(zip(repeat(region), rt[read]))
        seen.update(zip(repeat(region), names[read], rt[read]))
        return rt
    for region, k, (names, vals, nnz), per in (("intra4", 1, l4, 16), ("intra8", 2, l8, 4), ("intra16", 3, l4, 16)):
        read = np.repeat(kind == k, per)
        rt = tally(region, names, vals, nnz, read, k == 3)
        if k != 3:
            wraps = ec._first_pass_wraps if k == 1 else first_pass_wraps8
            seen["wrap%d" % (4 if k == 1 else 8)] += any(wraps(b) for b in vals[read & (rt == "full")][:200])
    chroma_read = np.repeat((kind != 0) & (rec["chroma_residual"] != 0), len(chroma_blocks))
    tally("chroma", *cb_, chroma_read, True)
    seen["untouched"] += int((np.repeat(kind == 0, 16) & l4[1].any(1)).sum() + (~chroma_read & cb_[1].any(1)).sum())
    co = np.where(owned, coeffs, ARENA_POISON).astype(np.int16) if bits == 8 else np.where(owned, coeffs * 32, 0x5A5A5A5A).astype(np.int32)
    return dict(rec=rec, coeffs=co, nnzc=nnzc, planes=picture(mb_w, mb_h, rng, bits, c422), seen=seen, slices=int(sl[-1]) + 1)


def matrix_cases(bits=8, c422=0):
    """the availability matrix: every size of SIZES with slices on / off and constrained_intra_pred on / off"""
    return {(w, h, s, c): intra_case(w, h, 1000 * w + 10 * h + 2 * s + c, s, c, bits, c422) for (w, h) in SIZES for (s, c) in VARIANTS}


def assert_coverage(seen):
    """the cases these pictures exist for, over the union of their Counters"""
    for tag in ("mode4", "mode8"):
        assert {k[1] for k in seen if k[0] == tag} == set(range(12)), (tag, sorted(k[1] for k in seen if k[0] == tag))
    for k in range(4):
        assert {p[2] for p in seen if p[:2] == ("tltr", k)} == TLTR8[k], (k, TLTR8[k])
    for key in ("tr_unavailable_4x4_block5", "tr_unavailable_8x8_block1", "tl_unavailable_8x8_block0", "top_unavailable_mid",
                ("plane_inter_topleft", "luma"), ("plane_inter_topleft", "chroma"), "dc128_mid", "wrap4", "wrap8", "untouched"):
        assert seen[key] > 0, key
    for region in ("intra4", "intra8", "intra16", "chroma"):
        for rt in ("full", "dc", "skip"):
            assert seen[region, rt] > 0, (region, rt)
    for region in ("intra4", "intra8"):
        assert seen[region, "single_ac", "full"] > 0 and seen[region, "dc_and_ac", "dc"] > 0 and seen[region, "dc_wrap", "full"] > 0
    assert seen["intra16", "dc_nnz0", "dc"] > 0 and seen["chroma", "dc_nnz0", "dc"] > 0 and seen["chroma", "dc_wrap", "full"] > 0
