"""Synthetic inputs shaped like the reference's own test generators (numpy, host side).

  lfg(seed, n)                 av_lfg_init + av_lfg_get stream      libavutil/lfg.c:30-46, lfg.h:40-43
  dct_test_blocks(test, n)     libavcodec/tests/dct.c:100-126 init_block() for the IDCT tests
  ref_fdct / ref_idct          libavcodec/dctref.c:58-122 (double precision, same summation order)
  dense_blocks(n)              uniform [-256,255] coefficients (SURVEY 8d config 2 (iii))
  yuv420p_frame(w, h, seed)    Y from the LFG first, then U[i], V[i] alternately, low byte of each draw
                               (the fill the survey probe used; CRC-pinned in tests/golden)
Used by tests/ and bench.py only; nothing here is on the product path.
"""
import hashlib
import struct

import numpy as np


def lfg(seed, n):
    """First n outputs of av_lfg_get() after av_lfg_init(seed) as uint32."""
    st = np.zeros(64, dtype=np.uint32)
    tmp = bytearray(16)
    for i in range(8, 64, 4):
        tmp[0:4] = struct.pack("<I", seed & 0xFFFFFFFF)
        tmp[4] = i
        tmp = bytearray(hashlib.md5(bytes(tmp)).digest())
        st[i:i + 4] = np.frombuffer(bytes(tmp), dtype="<u4")
    out = np.empty(n + 64, dtype=np.uint32)
    out[:64] = st
    k, total = 64, n + 64
    with np.errstate(over="ignore"):
        while k < total:
            m = min(24, total - k)          # x[k] = x[k-24] + x[k-55]; 24 outputs are independent
            out[k:k + m] = out[k - 24:k - 24 + m] + out[k - 55:k - 55 + m]
            k += m
    return out[64:]


def _dct_coefficients():
    c = np.zeros((8, 8), dtype=np.float64)
    for j in range(8):
        c[0, j] = np.sqrt(0.125)
        for i in range(1, 8):
            c[i, j] = 0.5 * np.cos((8 * i) * (j + 0.5) * np.pi / 64.0)
    return c


_COEF = _dct_coefficients()


def ref_fdct(blocks):
    """ff_ref_fdct on an (n, 8, 8) integer array -> int16, sequential-k accumulation like dctref.c:58-87."""
    b = blocks.astype(np.float64)
    n = b.shape[0]
    out = np.zeros((n, 8, 8), dtype=np.float64)
    for k in range(8):                       # out[i][j] = 8 * sum_k coef[i][k] * block[k][j]
        out += _COEF[None, :, k, None] * b[:, None, k, :]
    out *= 8
    res = np.zeros((n, 8, 8), dtype=np.float64)
    for k in range(8):                       # block[i][j] = sum_k out[i][k] * coef[j][k]
        res += out[:, :, k, None] * _COEF[None, None, :, k]
    return np.floor(res + 0.499999999999).astype(np.int64).astype(np.int16)


def ref_idct(blocks):
    """ff_ref_idct (dctref.c:96-122) on (n, 8, 8) -> int16."""
    b = blocks.astype(np.float64)
    n = b.shape[0]
    out = np.zeros((n, 8, 8), dtype=np.float64)
    for k in range(8):                       # out[i][j] = sum_k block[i][k] * coef[k][j]
        out += b[:, :, k, None] * _COEF[None, None, k, :]
    res = np.zeros((n, 8, 8), dtype=np.float64)
    for k in range(8):                       # block[i][j] = sum_k coef[k][i] * out[k][j]
        res += _COEF[None, k, :, None] * out[:, None, k, :]
    return np.floor(res + 0.5).astype(np.int64).astype(np.int16)


def dct_test_blocks(test, n, seed=1):
    """n blocks drawn exactly like NB_ITS calls of init_block(block, test, is_idct=1, prng) -> (n, 64) int16."""
    if test == 0:
        r = lfg(seed, 64 * n).reshape(n, 64)
        pix = (r % 512).astype(np.int64) - 256
        co = ref_fdct(pix.reshape(n, 8, 8)).astype(np.int32) >> 3
        return co.reshape(n, 64).astype(np.int16)
    if test == 1:
        # variable draws per block: j = r%10+1 then j x (value, position).  `block[lfg()%64] = lfg()%512-256`
        # leaves the draw order to the compiler; gcc evaluates the right-hand side first, and that order is
        # the one that reproduces fate-idct8x8's published statistics (tests/golden/fate_idct8x8.txt).
        r = lfg(seed, 21 * n + 64)
        out = np.zeros((n, 64), dtype=np.int16)
        p = 0
        for b in range(n):
            j = int(r[p] % 10) + 1
            p += 1
            for _ in range(j):
                val = int(r[p] % 512) - 256
                pos = int(r[p + 1] % 64)
                p += 2
                out[b, pos] = val
        return out
    if test == 2:
        r = lfg(seed, n)
        out = np.zeros((n, 64), dtype=np.int16)
        out[:, 0] = ((r % 4096).astype(np.int64) - 2048).astype(np.int16)
        out[:, 63] = (out[:, 0] & 1) ^ 1
        return out
    raise ValueError("test must be 0, 1 or 2")


def dense_blocks(n, seed=1):
    """Every coefficient uniform in [-256, 255]."""
    r = lfg(seed, 64 * n)
    return ((r % 512).astype(np.int64) - 256).astype(np.int16).reshape(n, 64)


def tile_large(base, n):
    """Repeat an (m, 64) block set up to n blocks with a cheap per-copy perturbation-free tiling (the
    distribution, not the exact stream, matters for throughput runs at 2^20 blocks)."""
    m = base.shape[0]
    reps = (n + m - 1) // m
    return np.tile(base, (reps, 1))[:n].copy()


def yuv420p_frame(w, h, seed=1):
    """(Y, U, V) uint8 planes, tight strides; chroma planes are ceil(w/2) x ceil(h/2)."""
    cw, ch = (w + 1) // 2, (h + 1) // 2
    r = lfg(seed, w * h + 2 * cw * ch)
    y = (r[:w * h] & 0xFF).astype(np.uint8).reshape(h, w)
    uv = (r[w * h:] & 0xFF).astype(np.uint8)
    u = uv[0::2].reshape(ch, cw).copy()
    v = uv[1::2].reshape(ch, cw).copy()
    return y, u, v


def pad_rows(plane, pad=8):
    """Copy a plane into rows of width+pad bytes whose padding repeats the last pixel (the byte the reference's
    fast-bilinear scaler reads past the end of each row); returns the strided view of the valid region."""
    h, w = plane.shape
    buf = np.empty((h, w + pad), dtype=plane.dtype)
    buf[:, :w] = plane
    buf[:, w:] = plane[:, -1:]
    return buf[:, :w]


def crc32_ieee_be(data):
    """av_crc(av_crc_get_table(AV_CRC_32_IEEE), 0, buf, len) (libavutil/crc.c): MSB-first CRC-32, polynomial
    0x04C11DB7, init 0, no final xor; av_crc keeps its state byte-swapped, so the value it returns is the
    byte-swapped register.  Chunk-parallel numpy evaluation (CRC with zero init is linear in the message)."""
    buf = np.frombuffer(bytes(data), dtype=np.uint8)
    tab = _crc_table()
    n = buf.size
    if n == 0:
        return 0
    chunks = max(1, min(4096, n // 64))
    clen = -(-n // chunks)
    pad = chunks * clen - n
    m = np.concatenate([np.zeros(pad, np.uint8), buf]).reshape(chunks, clen)   # leading zeros are neutral
    crc = np.zeros(chunks, dtype=np.uint32)
    for k in range(clen):
        crc = ((crc << np.uint32(8)) ^ tab[((crc >> np.uint32(24)) ^ m[:, k]) & 0xFF]).astype(np.uint32)
    # operator "append clen zero bytes" as four byte tables
    basis = (np.arange(256, dtype=np.uint32)[None, :] << (np.arange(4, dtype=np.uint32)[:, None] * 8)).astype(np.uint32).reshape(-1)
    for _ in range(clen):
        basis = ((basis << np.uint32(8)) ^ tab[(basis >> np.uint32(24)) & 0xFF]).astype(np.uint32)
    basis = basis.reshape(4, 256)
    acc = 0
    for c in crc.tolist():
        acc = int(basis[0][acc & 0xFF] ^ basis[1][(acc >> 8) & 0xFF] ^ basis[2][(acc >> 16) & 0xFF] ^ basis[3][acc >> 24]) ^ c
    return int.from_bytes(acc.to_bytes(4, "big"), "little")


_CRC_TAB = None


def _crc_table():
    global _CRC_TAB
    if _CRC_TAB is None:
        t = []
        for i in range(256):
            c = i << 24
            for _ in range(8):
                c = ((c << 1) ^ 0x04C11DB7) & 0xFFFFFFFF if c & 0x80000000 else (c << 1) & 0xFFFFFFFF
            t.append(c)
        _CRC_TAB = np.array(t, dtype=np.uint32)
    return _CRC_TAB


# ---------------------------------------------------------------------------------------------------
# H.264 synthetic macroblock work (SURVEY 8d config 3 shape): numpy structured arrays that match the record
# structs of include/avdsp_b200.h byte for byte.
# ---------------------------------------------------------------------------------------------------
RESIDUAL_DT = np.dtype([("luma_off", "<u4"), ("chroma_off", "<u4"), ("luma_mode", "u1"), ("chroma", "u1"), ("pad", "u1", (2,))])
MC_DT = np.dtype([("x", "<i2"), ("y", "<i2"), ("mvx", "<i2"), ("mvy", "<i2"), ("w", "u1"), ("h", "u1"), ("avg", "u1"), ("ref", "u1")])
WEIGHT_DT = np.dtype([("off", "<u4"), ("w", "u1"), ("h", "u1"), ("log2_denom", "u1"), ("pad", "u1"), ("weight", "<i2"),
                      ("weight_src", "<i2"), ("offset", "<i2"), ("pad2", "<i2")])
DEBLOCK_DT = np.dtype([("alpha", "u1", (2, 4)), ("beta", "u1", (2, 4)), ("tc0", "i1", (2, 4, 4)), ("intra", "u1", (2,)),
                       ("calpha", "u1", (2, 2, 2)), ("cbeta", "u1", (2, 2, 2)), ("ctc0", "i1", (2, 2, 2, 4)),
                       ("cintra", "u1", (2, 2)), ("pad", "u1", (2,))])
assert RESIDUAL_DT.itemsize == 12 and MC_DT.itemsize == 12 and WEIGHT_DT.itemsize == 16 and DEBLOCK_DT.itemsize == 104


def scan8(i):
    """libavcodec/h264dec.h:631-645"""
    plane, k = i >> 4, i & 15
    return 4 + (k & 1) + 2 * ((k >> 2) & 1) + 8 * (1 + ((k >> 1) & 1) + 2 * (k >> 3) + 5 * plane)


def h264_picture(mb_w, mb_h, seed=1):
    """Random 4:2:0 picture planes (tight strides, 16*mb_w x 16*mb_h)."""
    w, h = 16 * mb_w, 16 * mb_h
    r = lfg(seed, w * h * 3 // 2)
    y = (r[:w * h] & 0xFF).astype(np.uint8).reshape(h, w)
    cb = (r[w * h:w * h + w * h // 4] & 0xFF).astype(np.uint8).reshape(h // 2, w // 2)
    cr = (r[w * h + w * h // 4:] & 0xFF).astype(np.uint8).reshape(h // 2, w // 2)
    return y, cb, cr


def h264_residual_work(mb_w, mb_h, seed=2, p_coded=0.5, modes=(0, 1, 2)):
    """Per-MB residual records, the reference-layout coefficient buffer (n, 768) int16 and nnzc (n, 120) u8."""
    rng = np.random.default_rng(seed)
    n = mb_w * mb_h
    rec = np.zeros(n, dtype=RESIDUAL_DT)
    mbx, mby = np.arange(n) % mb_w, np.arange(n) // mb_w
    rec["luma_off"] = mby * 16 * (16 * mb_w) + mbx * 16
    rec["chroma_off"] = mby * 8 * (8 * mb_w) + mbx * 8
    rec["luma_mode"] = rng.choice(np.array(modes, dtype=np.uint8), size=n)
    rec["chroma"] = rng.integers(0, 2, size=n)
    coeffs = np.zeros((n, 768), dtype=np.int16)
    nnzc = np.zeros((n, 120), dtype=np.uint8)
    for m in range(n):
        mode = int(rec["luma_mode"][m])
        blocks = list(range(0, 16, 4)) if mode == 2 else list(range(16))
        size = 64 if mode == 2 else 16
        for i in blocks + [16, 17, 18, 19, 32, 33, 34, 35]:
            sz = size if i < 16 else 16
            kind = rng.integers(0, 4) if rng.random() < p_coded * 1.5 else 0      # 0 none, 1 dc only (nnz 0), 2 dc (nnz 1), 3 full
            if kind == 0:
                continue
            if kind in (1, 2):
                coeffs[m, 16 * i] = rng.integers(-2000, 2000)
                nnzc[m, scan8(i)] = 0 if kind == 1 else 1
            else:
                coeffs[m, 16 * i:16 * i + sz] = rng.integers(-300, 300, size=sz)
                nnzc[m, scan8(i)] = rng.integers(2, 17)
    return rec, coeffs, nnzc


def h264_mc_work(mb_w, mb_h, seed=3, max_mv=64, nrefs=2, avg_second=True):
    """One record per 8x8 / 16x8 / 8x16 / 16x16 / 4x4 partition, covering every MB exactly once with `put`, plus an
    `avg` second direction on some partitions.  Vectors may leave the picture (edge replication is exercised)."""
    rng = np.random.default_rng(seed)
    out = []
    for mby in range(mb_h):
        for mbx in range(mb_w):
            shape = rng.integers(0, 5)
            parts = {0: [(0, 0, 16, 16)], 1: [(0, 0, 16, 8), (0, 8, 16, 8)], 2: [(0, 0, 8, 16), (8, 0, 8, 16)],
                     3: [(x, y, 8, 8) for y in (0, 8) for x in (0, 8)],
                     4: [(x, y, 4, 4) for y in range(0, 16, 4) for x in range(0, 16, 4)]}[int(shape)]
            for (px, py, w, h) in parts:
                mv = rng.integers(-max_mv, max_mv + 1, size=2)
                out.append((16 * mbx + px, 16 * mby + py, mv[0], mv[1], w, h, 0, rng.integers(0, nrefs)))
                if avg_second and rng.random() < 0.3:
                    mv = rng.integers(-max_mv, max_mv + 1, size=2)
                    out.append((16 * mbx + px, 16 * mby + py, mv[0], mv[1], w, h, 1, rng.integers(0, nrefs)))
    rec = np.zeros(len(out), dtype=MC_DT)
    for k, name in enumerate(("x", "y", "mvx", "mvy", "w", "h", "avg", "ref")):
        rec[name] = [o[k] for o in out]
    return rec


def h264_deblock_work(mb_w, mb_h, seed=4, slices=1):
    """Random per-edge parameters in the ranges of the reference's alpha/beta/tc0 tables
    (libavcodec/h264_loopfilter.c:40-101).  Picture-boundary edges (and slice-boundary edges when slices > 1,
    disable_deblocking_filter_idc = 2) carry alpha = 0."""
    rng = np.random.default_rng(seed)
    n = mb_w * mb_h
    rec = np.zeros(n, dtype=DEBLOCK_DT)
    rec["alpha"] = rng.integers(0, 120, size=(n, 2, 4))
    rec["beta"] = rng.integers(0, 19, size=(n, 2, 4))
    rec["tc0"] = rng.integers(-1, 10, size=(n, 2, 4, 4))
    rec["intra"] = rng.integers(0, 2, size=(n, 2))                   # only edge 0 may be intra
    rec["calpha"] = rng.integers(0, 120, size=(n, 2, 2, 2))
    rec["cbeta"] = rng.integers(0, 19, size=(n, 2, 2, 2))
    rec["ctc0"] = rng.integers(0, 11, size=(n, 2, 2, 2, 4))
    rec["cintra"] = rng.integers(0, 2, size=(n, 2, 2))
    per = -(-n // slices)
    for m in range(n):
        mbx, mby = m % mb_w, m // mb_w
        first_in_slice = (m % per) == 0
        left_other = mbx == 0 or (slices > 1 and first_in_slice)
        top_other = mby == 0 or (slices > 1 and (m - mb_w) // per != m // per)
        if left_other:
            rec["alpha"][m, 0, 0] = 0
            rec["calpha"][m, :, 0, 0] = 0
        if top_other:
            rec["alpha"][m, 1, 0] = 0
            rec["calpha"][m, :, 1, 0] = 0
    return rec


# ---- decoder side information for the deblocking-decision kernel (the reference's own array layouts) ----
MB_INTRA4x4, MB_INTRA16x16, MB_INTRA_PCM, MB_16x16, MB_16x8, MB_8x16, MB_8x8 = 1, 2, 4, 8, 16, 32, 64
MB_DIRECT2, MB_SKIP, MB_P0L0, MB_P1L0, MB_P0L1, MB_P1L1, MB_8x8DCT = 0x100, 0x800, 0x1000, 0x2000, 0x4000, 0x8000, 0x01000000
H264_CHROMA_QP = np.array(list(range(30)) + [29, 30, 31, 32, 32, 33, 34, 34, 35, 35, 36, 36, 37, 37, 37, 38, 38, 38, 39, 39, 39, 39], np.uint8)


def h264_chroma_qp_table(bit_depth, offset):
    """One row of PPS.chroma_qp_table in the decoder's QP' scale: QP'c for QP'y = 0..max_qp (max_qp = 51 + qp_bd_offset) and
    chroma_qp_index_offset `offset`.  The standard's qPI = Clip3(-QpBdOffsetC, 51, QPy + offset) maps to QPc through H264_CHROMA_QP
    (identity below 30, so also for the negative qPI of 9 / 10 bit), and QP'c = QPc + QpBdOffsetC.  Entries past max_qp stay 0."""
    bd = 6 * (bit_depth - 8)
    max_qp = 51 + bd
    qpi = np.clip(np.arange(max_qp + 1) + offset, 0, max_qp) - bd
    row = np.zeros(64, np.uint8)
    row[:max_qp + 1] = np.where(qpi < 0, qpi, H264_CHROMA_QP[np.maximum(qpi, 0)]) + bd
    return row


def h264_deblock_info(mb_w, mb_h, seed=5, n_slices=3, bipred=False, cabac=1, t8x8=0, mode=1, qp_lo=10, qp_hi=51,
                      p_intra=0.15, cb_off=0, cr_off=0, bit_depth=8):
    """Random but self-consistent side information of one progressive picture, in the layouts libavcodec keeps it
    (H264Picture.mb_type / qscale_table / motion_val / ref_index, H264Context.non_zero_count / cbp_table /
    slice_table / ref2frm, PPS.chroma_qp_table): what ff_h264_deblock_params_cuda and the oracle consume.
    Motion vectors differ by 0..8 quarter-pels between partitions so the |d| >= 4 rule is exercised both ways.
    bit_depth 9 / 10: qscale_table, chroma_qp_table and qp_thresh in the decoder's QP' scale (0..max_qp, max_qp = 51 + 6 * (bit_depth - 8),
    h264_cavlc.c:1094, h264_ps.c:662, h264_slice.c:1815-1820), drawn from a second random stream after the 8-bit draws: qscale weighted
    towards both ends -- 0 (some of those macroblocks I_PCM, which the decoder stores with qscale 0, h264_cavlc.c:782), the slice's
    qp_thresh +- 2 and max_qp -- and otherwise uniform over [qp_lo, qp_hi] + qp_bd_offset; alpha / beta offsets over -12..12; unless
    cb_off / cr_off are given, two different chroma_qp_index_offsets in -12..12."""
    r = np.random.RandomState(seed)
    ms, bs = mb_w + 1, 4 * mb_w
    n = ms * mb_h
    d = {"mb_w": mb_w, "mb_h": mb_h, "cabac": cabac, "t8x8": t8x8, "n_slices": n_slices}
    mb_type = np.zeros(n, np.uint32); qp = np.zeros(n, np.int8); nnz = np.zeros((n, 48), np.uint8)
    cbp = np.zeros(n, np.uint16); sl = np.full(n, 0xFFFF, np.uint16)
    mv = np.zeros((2, 4 * mb_h, bs, 2), np.int16); ref = np.full((2, n, 4), -1, np.int8)
    per = -(-mb_w * mb_h // n_slices)
    for y in range(mb_h):
        for x in range(mb_w):
            xy = x + y * ms
            sl[xy] = (x + y * mb_w) // per
            qp[xy] = r.randint(qp_lo, qp_hi + 1)
            dct8 = MB_8x8DCT if (t8x8 and r.rand() < 0.4) else 0
            if r.rand() < p_intra:
                mb_type[xy] = (MB_INTRA4x4 | dct8) if r.rand() < 0.6 else MB_INTRA16x16
                nnz[xy, :16] = r.randint(0, 17, 16)
                cbp[xy] = r.randint(0, 16) | (r.randint(0, 16) << 12)
                continue
            part = [MB_16x16, MB_16x8, MB_8x16, MB_8x8][r.randint(0, 4)]
            if bipred:
                use = [[1, 0], [0, 1], [1, 1]][r.randint(0, 3)]
                if r.rand() < 0.1: use = [1, 1]
            else:
                use = [1, 0]
            t = part | dct8
            if use[0]: t |= MB_P0L0 | MB_P1L0
            if use[1]: t |= MB_P0L1 | MB_P1L1
            if part == MB_16x16 and r.rand() < 0.2: t |= MB_SKIP
            if bipred and r.rand() < 0.1: t |= MB_DIRECT2
            mb_type[xy] = t
            # partition geometry in 4x4 units
            rects = {MB_16x16: [(0, 0, 4, 4)], MB_16x8: [(0, 0, 4, 2), (0, 2, 4, 2)], MB_8x16: [(0, 0, 2, 4), (2, 0, 2, 4)],
                     MB_8x8: [(0, 0, 2, 2), (2, 0, 2, 2), (0, 2, 2, 2), (2, 2, 2, 2)]}[part]
            base = r.randint(-6, 7, 2)
            for l in range(2):
                if not use[l]:
                    continue
                for (bx, by, bw, bh) in rects:
                    ri = r.randint(0, 3)
                    if part == MB_8x8 and r.rand() < 0.5:                       # sub-partitions: per-4x4 vectors
                        for yy in range(by, by + bh):
                            for xx in range(bx, bx + bw):
                                mv[l, 4 * y + yy, 4 * x + xx] = base + r.randint(0, 6, 2)
                    else:
                        mv[l, 4 * y + by:4 * y + by + bh, 4 * x + bx:4 * x + bx + bw] = base + r.randint(0, 6, 2)
                    for yy in range(by // 2, (by + bh + 1) // 2):
                        for xx in range(bx // 2, (bx + bw + 1) // 2):
                            ref[l, xy, xx + 2 * yy] = ri
            coded = r.rand(4) < 0.45                                              # per 8x8 luma
            for k in range(16):
                b8 = ((k & 3) >> 1) + 2 * (k >> 3)
                nnz[xy, k] = r.randint(1, 17) if (coded[b8] and r.rand() < 0.6) else 0
            c = 0
            for b8 in range(4):
                if nnz[xy, [b8 % 2 * 2 + b8 // 2 * 8 + o for o in (0, 1, 4, 5)]].any(): c |= 1 << b8
            cbp[xy] = c | (r.randint(0, 3) << 4) | ((r.randint(0, 16) << 12) if dct8 else 0)
    # per-slice parameters: {alpha_c0_offset, beta_offset, deblocking_filter, list_count, qp_thresh, ref2frm[2][64]}
    sp = np.zeros((n_slices, 133), np.int32)
    for s in range(n_slices):
        a, b = 2 * r.randint(-3, 4), 2 * r.randint(-3, 4)
        r2f = np.full((2, 64), -1, np.int32)
        ids = r.permutation(6)
        for l in range(2):
            for i in range(4):
                r2f[l, 2 + i] = 4 * int(ids[(i + 2 * l) % 4 if bipred else i % 3]) + 3      # some indices share a frame
        sp[s, :5] = [a, b, mode, 2 if bipred else 1, 15 - min(a, b) - max(0, cb_off, cr_off)]
        sp[s, 5:] = r2f.reshape(-1)
    if bit_depth != 8:
        if bit_depth not in (9, 10):
            raise ValueError("bit_depth 8, 9 or 10")
        h = np.random.RandomState(seed + 1000 * bit_depth)
        bd = 6 * (bit_depth - 8)
        max_qp = 51 + bd
        if cb_off == 0 and cr_off == 0:
            cb_off, cr_off = (int(v) for v in h.choice(np.arange(-12, 13), 2, replace=False))
        for s in range(n_slices):
            a, b = 2 * h.randint(-6, 7), 2 * h.randint(-6, 7)
            sp[s, :5] = [a, b, mode, 2 if bipred else 1, 15 - min(a, b) - max(0, cb_off, cr_off) + bd]
        for y in range(mb_h):
            for x in range(mb_w):
                xy = x + y * ms
                u = h.rand()
                if u < 0.1:
                    qp[xy] = 0
                    if h.rand() < 0.5:
                        mb_type[xy] = MB_INTRA_PCM
                        nnz[xy] = 16
                elif u < 0.2:
                    qp[xy] = max_qp
                elif u < 0.45:
                    qp[xy] = np.clip(sp[sl[xy], 4] + h.randint(-2, 3), 0, max_qp)
                else:
                    qp[xy] = h.randint(min(qp_lo + bd, max_qp), min(qp_hi + bd, max_qp) + 1)
    cqt = np.zeros((2, 64), np.uint8)
    for t, off in enumerate((cb_off, cr_off)):
        cqt[t] = h264_chroma_qp_table(bit_depth, off)
    d.update(bit_depth=bit_depth, mb_type=mb_type, qscale=qp, nnz=nnz, cbp=cbp, slice_table=sl, mv0=np.ascontiguousarray(mv[0]), mv1=np.ascontiguousarray(mv[1]),
             ref0=np.ascontiguousarray(ref[0]), ref1=np.ascontiguousarray(ref[1]), slice_params=sp, chroma_qp_table=cqt)
    return d


INTRA_DT = np.dtype([("kind", "u1"), ("mode16", "u1"), ("chroma_mode", "u1"), ("chroma_residual", "u1"), ("mode4", "u1", (16,)),
                     ("topleft", "<u2"), ("topright", "<u2")])


def h264_intra_work(mb_w, mb_h, seed=8, p_intra=1.0, p_coded=0.5):
    """Intra macroblocks of one single-slice picture the way the decoder hands them to hl_decode_mb(): prediction modes
    already substituted for what is available (check_intra4x4_pred_mode / check_intra_pred_mode, h264_parse.c), the
    sample-availability masks of fill_decode_caches (h264_mvpred.h:468-508), coefficients in the sl->mb layout with
    their non_zero_count_cache.  Returns (records, coeffs int16 [n][768], nnzc uint8 [n][120])."""
    r = np.random.RandomState(seed)
    n = mb_w * mb_h
    rec = np.zeros(n, INTRA_DT)
    coeffs = np.zeros((n, 768), np.int16)
    nnzc = np.zeros((n, 120), np.uint8)

    def fill_block(m, i, size):
        """coefficients of 4x4 block i (size 16) or 8x8 block i (size 64, stored at i * 16): nnz in {0, 1 (DC), many}"""
        u = r.rand()
        if u > p_coded:
            return 0
        if u < p_coded / 3:
            coeffs[m, 16 * i] = r.randint(-800, 801) or 64
            return 1
        coeffs[m, 16 * i:16 * i + size] = (r.randint(-64, 65, size) * (r.rand(size) < 0.4)).astype(np.int16) * 4
        coeffs[m, 16 * i] = r.randint(-600, 601)
        return 16

    for y in range(mb_h):
        for x in range(mb_w):
            m = x + y * mb_w
            if r.rand() >= p_intra:
                continue
            top, left = y > 0, x > 0
            tl_mb, tr_mb = top and left, top and x + 1 < mb_w
            topleft, topm, leftm, topright = 0xFFFF, 0xFFFF, 0xFFFF, 0xEEEA
            if not top:
                topleft, topm, topright = 0xB3FF, 0x33FF, 0x26EA
            if not left:
                topleft &= 0xDF5F; leftm &= 0x5F5F
            if not tl_mb:
                topleft &= 0x7FFF
            if not tr_mb:
                topright &= 0xFBFF
            rec["topleft"][m], rec["topright"][m] = topleft, topright
            kind = r.randint(1, 4)
            rec["kind"][m] = kind

            def big_mode(t, l):
                ok = [0] + ([2] if t else []) + ([1] if l else []) + ([3] if t and l else [])
                md = ok[r.randint(0, len(ok))]
                if md == 0:
                    md = 0 if (t and l) else 4 if l else 5 if t else 6
                return md
            rec["chroma_mode"][m] = big_mode(top, left)
            rec["chroma_residual"][m] = r.rand() < 0.7
            if kind == 3:
                rec["mode16"][m] = big_mode(top, left)
                for i in range(16):
                    nnzc[m, scan8(i)] = fill_block(m, i, 16)
                    if nnzc[m, scan8(i)] == 1:                 # add16intra treats "DC only" as nnz 0 + DC (the DC comes from the luma DC transform)
                        nnzc[m, scan8(i)] = 0
            else:
                step = 1 if kind == 1 else 4
                for i in range(0, 16, step):
                    t = bool(topm & (0x8000 >> i)); l = bool(leftm & (0x8000 >> i))
                    ok = [2] + ([0, 3, 7] if t else []) + ([1, 8] if l else []) + ([4, 5, 6] if t and l else [])
                    md = ok[r.randint(0, len(ok))]
                    if md == 2:
                        md = 2 if (t and l) else 9 if l else 10 if t else 11
                    rec["mode4"][m, i] = md
                    nz = fill_block(m, i, 16 if kind == 1 else 64)
                    if kind == 1:
                        nnzc[m, scan8(i)] = nz
                    else:
                        for k in range(4):
                            nnzc[m, scan8(i + k)] = nz
            if rec["chroma_residual"][m]:
                for i in list(range(16, 20)) + list(range(32, 36)):
                    nz = fill_block(m, i, 16)
                    nnzc[m, scan8(i)] = 0 if nz == 1 else nz
    return rec, coeffs, nnzc


def zigzag_scan_tables():
    """(permutated, raster_end) of the 8x8 zigzag scan for an IDCT without coefficient permutation -- what
    ff_init_scantable (libavcodec/idctdsp.c:28-47) builds from ff_zigzag_direct: walk the anti-diagonals, even ones
    upwards (towards the top right), odd ones downwards."""
    order = []
    for d in range(15):
        cells = [(d - x, x) for x in range(8) if 0 <= d - x < 8]          # (row, col), col ascending = walking up-right
        if d % 2 == 1:
            cells.reverse()
        order += [r * 8 + c for r, c in cells]
    perm = np.array(order, np.uint8)
    return perm, np.maximum.accumulate(perm).astype(np.uint8)


MECMP_DT = np.dtype([("cur_off", "<u4"), ("ref_off", "<u4")])
HPEL_DT = np.dtype([("dst_off", "<u4"), ("src_off", "<u4"), ("tab", "u1"), ("sidx", "u1"), ("dxy", "u1"), ("h", "u1")])
assert MECMP_DT.itemsize == 8 and HPEL_DT.itemsize == 12


def me_frames(w, h, seed=1, shift=(3, -5), noise=3):
    """cur / ref luma planes for the motion-search workload: ref from the LFG, cur = ref shifted by `shift` plus small
    noise (so the arg-min is meaningful), as SURVEY 8d config 4 asks."""
    ref = (lfg(seed, w * h) & 0xFF).astype(np.uint8).reshape(h, w)
    rng = np.random.default_rng(seed)
    cur = np.roll(ref, shift, axis=(0, 1)).astype(np.int64) + rng.integers(-noise, noise + 1, size=(h, w))
    return np.clip(cur, 0, 255).astype(np.uint8), ref


def h264_config3_picture(mb_w=120, mb_h=68, slices=64, seed=0):
    """BASELINE config 3, one synthetic P picture: two reference pictures, quarter-pel MC records for every partition, residual
    records + coefficient arena, per-edge deblocking records with `slices` slices (disable_deblocking_filter_idc = 2: no edge crosses
    a slice), and mc_first[m] = index of macroblock m's first MC record (records are in macroblock raster order)."""
    refs = [h264_picture(mb_w, mb_h, seed=11 + seed), h264_picture(mb_w, mb_h, seed=12 + seed)]
    mc = h264_mc_work(mb_w, mb_h, seed=5 + seed)
    res, coeffs, nnzc = h264_residual_work(mb_w, mb_h, seed=6 + seed)
    dbk = h264_deblock_work(mb_w, mb_h, seed=7 + seed, slices=slices)
    mb_of = (mc["y"].astype(np.int64) // 16) * mb_w + mc["x"].astype(np.int64) // 16
    assert np.all(np.diff(mb_of) >= 0)
    mc_first = np.searchsorted(mb_of, np.arange(mb_w * mb_h + 1)).astype(np.uint32)
    return dict(mb_w=mb_w, mb_h=mb_h, slices=slices, refs=refs, mc=mc, mc_first=mc_first, res=res, coeffs=coeffs, nnzc=nnzc, dbk=dbk)
