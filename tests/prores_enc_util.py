"""TEST INFRASTRUCTURE.  ProRes encoder cases for tests/test_prores_enc_cpu.py, tests/test_gpu_prores_enc.py and tools/prores_enc_bench.py:
seeded source frames, the options of each case, the product's call (host-compiled or on the GPU) and the reference encoder
(oracle/_ref/libproresencref.so), and a packet parser that reads back what a packet says about its slices."""
import ctypes as C
import itertools

import numpy as np

from libav_b200 import tables
import prores_util as PU

vp, i32 = C.c_void_p, C.c_int
FMT_422, FMT_444, FMT_4444 = 0, 1, 2


class Opts(C.Structure):        # oracle/refbuild/refapi_prores_enc.c RefProresEncOpts
    _fields_ = [("fmt", C.c_int32), ("interlaced", C.c_int32), ("profile", C.c_int32), ("mbs_per_slice", C.c_int32),
                ("bits_per_mb", C.c_int32), ("quant_sel", C.c_int32), ("alpha_bits", C.c_int32), ("force_quant", C.c_int32),
                ("vendor", C.c_char * 4), ("color_primaries", C.c_uint8), ("color_trc", C.c_uint8), ("colorspace", C.c_uint8),
                ("reserved", C.c_uint8)]


def ref():
    """the reference encoder library with prototypes, or None when oracle/_ref was not built"""
    from oracle import loader
    lib = loader.ref_lib("proresenc")
    if lib is None:
        return None
    lib.ref_prores_encode_opts.restype = i32
    lib.ref_prores_encode_opts.argtypes = [C.POINTER(Opts), i32, i32, vp, vp, vp, i32, vp, i32]
    lib.ref_prores_enc_tables.restype, lib.ref_prores_enc_tables.argtypes = i32, [vp]
    lib.ref_prores_encode_frames.restype = i32
    lib.ref_prores_encode_frames.argtypes = [C.POINTER(Opts), i32, i32, i32, vp, vp, vp, i32, vp, i32]
    return lib


class Case:
    """one frame and its options.  content: 'natural' (prores_util.source_frame), 'noise', 'flat', 'extremes'; alpha: 'natural',
    'runs' (runs below and above 16 and diffs at +-dsize), 'noise'"""

    def __init__(self, fmt, w, h, interlaced=0, profile=2, mbs_per_slice=8, bits_per_mb=0, quant_sel=-1, alpha_bits=16, force_quant=0,
                 vendor=b"Lavc", colour=(2, 2, 2), content="natural", alpha="natural", seed=1, pad=0):
        self.fmt, self.w, self.h, self.interlaced, self.profile = fmt, w, h, interlaced, profile
        self.mbs_per_slice, self.bits_per_mb, self.quant_sel, self.alpha_bits, self.force_quant = mbs_per_slice, bits_per_mb, quant_sel, alpha_bits, force_quant
        self.vendor, self.colour, self.content, self.alpha, self.seed, self.pad = vendor, colour, content, alpha, seed, pad
        self.planes = frame(fmt, w, h, content, alpha, seed)

    def __repr__(self):
        return "Case(fmt=%d %dx%d il=%d prof=%d mps=%d bpm=%d qs=%d ab=%d fq=%d %s/%s seed=%d)" % (
            self.fmt, self.w, self.h, self.interlaced, self.profile, self.mbs_per_slice, self.bits_per_mb, self.quant_sel,
            self.alpha_bits, self.force_quant, self.content, self.alpha, self.seed)

    @property
    def abits(self):
        return self.alpha_bits if self.fmt == FMT_4444 else 0

    def opts(self):
        return Opts(fmt=self.fmt, interlaced=self.interlaced, profile=self.profile, mbs_per_slice=self.mbs_per_slice,
                    bits_per_mb=self.bits_per_mb, quant_sel=self.quant_sel, alpha_bits=self.alpha_bits, force_quant=self.force_quant,
                    vendor=self.vendor, color_primaries=self.colour[0], color_trc=self.colour[1], colorspace=self.colour[2])

    def linesizes(self):
        return [p.shape[1] * 2 + self.pad if p is not None else 0 for p in self.planes]

    def work(self, ptrs, out, cap, out_size):
        w = tables.FFProresEncodeWork()
        for p in range(4):
            w.data[p] = ptrs[p] or 0
        for p, ls in enumerate(self.linesizes()):
            w.linesize[p] = ls
        w.width, w.height, w.pix_fmt, w.interlaced, w.profile = self.w, self.h, self.fmt, self.interlaced, self.profile
        w.mbs_per_slice, w.bits_per_mb, w.quant_sel, w.alpha_bits, w.force_quant = self.mbs_per_slice, self.bits_per_mb, self.quant_sel, self.alpha_bits, self.force_quant
        w.vendor = self.vendor
        w.color_primaries, w.color_trc, w.colorspace = self.colour
        w.out, w.out_capacity, w.out_size = out, cap, out_size
        return w

    def padded(self, p):
        """plane p laid out at this case's linesize (bytes), as uint8"""
        a = self.planes[p]
        if a is None:
            return None
        ls = self.linesizes()[p]
        buf = np.full((a.shape[0], ls), 0xAB, np.uint8)
        buf[:, :a.shape[1] * 2] = a.view(np.uint8).reshape(a.shape[0], -1)
        return buf

    def capacity(self):
        mbw = (self.w + 15) // 16
        mbh = (self.h + 15) // 16 + 1
        return 4096 + mbw * mbh * 16 * 16 * 4 * 4 + (mbw * mbh * 256 * 3 if self.abits else 0)


def frame(fmt, w, h, content, alpha, seed):
    """the four planes (alpha None unless 4:4:4:4) as uint16 arrays"""
    r = np.random.default_rng(seed)
    cw = w if fmt != FMT_422 else (w + 1) // 2
    if content == "natural":
        planes = PU.source_frame(fmt, w, h, seed)[:3]
    elif content == "noise":
        planes = [r.integers(0, 1024, (h, pw)).astype(np.uint16) for pw in (w, cw, cw)]
    elif content == "flat":
        planes = [np.full((h, pw), v, np.uint16) for pw, v in ((w, int(r.integers(0, 1024))), (cw, 512), (cw, int(r.integers(0, 1024))))]
    elif content == "extremes":
        planes = [(r.integers(0, 2, (h, pw)) * 1023).astype(np.uint16) for pw in (w, cw, cw)]
    else:
        raise ValueError(content)
    a = None
    if fmt == FMT_4444:
        if alpha == "natural":
            a = PU.source_frame(FMT_4444, w, h, seed + 100)[3]
        elif alpha == "noise":
            a = r.integers(0, 1024, (h, w)).astype(np.uint16)
        elif alpha == "runs":
            # runs of 1..40 samples (below and above 16) of values whose steps, in the coded units, include +-dsize and +-(dsize + 1)
            # (8 and 9 at 8 bits: source steps of 32 and 36; 64 and 65 at 16 bits: source steps of 1) and larger ones
            flat = []
            v = 512
            while len(flat) < w * h:
                step = int(r.choice([0, 1, -1, 4, -4, 32, -32, 36, -36, 1, 2, 16, -16, 17, -17, 300, -300]))
                v = min(max(v + step, 0), 1023)
                flat += [v] * int(r.choice([1, 2, 3, 15, 16, 17, 40]))
            a = np.array(flat[:w * h], np.uint16).reshape(h, w)
        else:
            raise ValueError(alpha)
    return [np.ascontiguousarray(p) for p in planes] + [a]


def ref_encode(lib, case):
    """the reference's packet and each slice's quantiser"""
    planes = [case.padded(p) for p in range(4)]
    ptrs = (C.c_void_p * 4)(*[p.ctypes.data if p is not None else None for p in planes])
    ls = (C.c_int * 4)(*case.linesizes())
    cap = case.capacity()
    out = np.zeros(cap, np.uint8)
    sq = np.zeros(1 << 16, np.int32)
    n = lib.ref_prores_encode_opts(C.byref(case.opts()), case.w, case.h, ptrs, ls, PU.P(out), cap, PU.P(sq), len(sq))
    assert n > 0, ("reference encode failed", case, n)
    return out[:n].copy(), sq


def run(lib, mem, cases, cap_delta=None, stream=None):
    """ff_prores_encode_frames_cuda over the cases in one call: (rc, packets, out_sizes, raw output buffers).  cap_delta: out_capacity =
    (the reference's packet size + cap_delta) for each case, given as a list of (size, delta)"""
    works, outs, sizes = [], [], []
    for k, c in enumerate(cases):
        ptrs = [mem.put(c.padded(p)) if c.planes[p] is not None else None for p in range(4)]
        cap = c.capacity() if cap_delta is None else cap_delta[k][0] + cap_delta[k][1]
        o = mem.put(np.full(cap + 64, 0xCD, np.uint8))
        z = mem.put(np.zeros(1, np.int32))
        outs.append((o, cap)); sizes.append(z)
        works.append(c.work(ptrs, o, cap, z))
    arr = (tables.FFProresEncodeWork * len(works))(*works)
    need = lib.ff_prores_encode_workspace_cuda(arr, len(works))
    ws = mem.put(np.zeros(max(need, 1), np.uint8))
    rc = lib.ff_prores_encode_frames_cuda(arr, len(works), C.c_void_p(ws), need, stream)
    mem.sync()
    got_sizes = [int(mem.get(z, np.int32, (1,))[0]) for z in sizes]
    raws = [mem.get(o, np.uint8, (cap + 64,)) for o, cap in outs]
    pkts = [r[:s].copy() if s > 0 else None for r, s in zip(raws, got_sizes)]
    return rc, pkts, got_sizes, raws


def slice_quants(pkt):
    """each slice's quantiser as the packet says, pictures in order"""
    hsize = int(pkt[8]) << 8 | int(pkt[9])
    pos = 8 + hsize
    interlaced = (pkt[20] >> 2) & 3
    qs = []
    for _ in range(2 if interlaced else 1):
        ph = int(pkt[pos]) >> 3
        ns = int(pkt[pos + 5]) << 8 | int(pkt[pos + 6])
        idx = pos + ph
        data = idx + 2 * ns
        for s in range(ns):
            qs.append(int(pkt[data + 1]))
            data += int(pkt[idx + 2 * s]) << 8 | int(pkt[idx + 2 * s + 1])
        pos = data
    return qs


def compare(case, got, want, want_q):
    """byte-identical packets; on a difference, the first slice whose quantiser differs, or the first differing byte"""
    if got is not None and np.array_equal(got, want):
        return
    msg = [repr(case), "sizes %s vs %d" % (None if got is None else len(got), len(want))]
    if got is not None:
        q = slice_quants(got)
        wq = list(want_q[:len(q)])
        bad = [i for i, (a, b) in enumerate(zip(q, wq)) if a != b]
        if bad:
            msg.append("first slice with another quantiser: %d (%d vs %d)" % (bad[0], q[bad[0]], wq[bad[0]]))
        n = min(len(got), len(want))
        d = np.flatnonzero(got[:n] != want[:n])
        msg.append("first differing byte: %s" % (d[0] if len(d) else n))
    raise AssertionError("; ".join(msg))


def pairwise(values):
    """a small set of rows in which every pair of values of any two of the lists occurs together (greedy covering)"""
    need = set()
    for i, j in itertools.combinations(range(len(values)), 2):
        for a in values[i]:
            for b in values[j]:
                need.add((i, a, j, b))
    rows = []
    allrows = list(itertools.product(*values))
    rng = np.random.default_rng(7)
    order = rng.permutation(len(allrows))
    while need:
        best, gain = None, -1
        for k in order:
            row = allrows[k]
            g = sum((i, row[i], j, row[j]) in need for i, j in itertools.combinations(range(len(row)), 2))
            if g > gain:
                best, gain = row, g
        rows.append(best)
        for i, j in itertools.combinations(range(len(best)), 2):
            need.discard((i, best[i], j, best[j]))
    return rows


def matrix_cases():
    """formats x profiles x field order x mbs_per_slice, pairwise; sizes vary with the row so that right-edge slices of every width occur"""
    rows = pairwise([[FMT_422, FMT_444, FMT_4444], [0, 1, 2, 3, 4], [0, 1, 2], [1, 2, 4, 8]])
    sizes = [(112, 48), (200, 40), (72, 66), (184, 96), (120, 35), (40, 51), (88, 32), (136, 64), (24, 16)]
    cases = []
    for k, (fmt, prof, il, mps) in enumerate(rows):
        w, h = sizes[k % len(sizes)]
        if il and h // 2 <= 16 * ((h + 31) // 32 - 1):
            h += 2
        cases.append(Case(fmt, w, h, il, prof, mps, seed=100 + k))
    return cases


def edge_cases():
    """widths 16k, 16k + 1 (the zero 4:2:2 chroma block), 16k + 2, 16k + 9 and 1; right-edge slices of 4, 2, 1 macroblocks; heights 16k + 1
    and interlaced 32k + 3, 32k + 17, 32k + 31"""
    cs = []
    for k, w in enumerate((64, 65, 66, 73, 1, 17, 9, 2)):
        cs.append(Case(FMT_422, w, 20, 0, 3, 8, seed=200 + k))
    for k, w in enumerate((65, 73, 1)):
        cs.append(Case(FMT_444, w, 18, 0, 2, 4, seed=210 + k))
        cs.append(Case(FMT_4444, w, 18, 2, 4, 2, seed=220 + k))
    for k, w in enumerate((16 * 15, 16 * 14, 16 * 13, 16 * 7)):                     # last slices 4 + 2 + 1, 4 + 2, 4 + 1, 4 + 2 + 1
        cs.append(Case(FMT_422, w, 32, 0, 1, 8, seed=230 + k))
    for k, h in enumerate((17, 33, 49, 1)):
        cs.append(Case(FMT_422, 48, h, 0, 2, 2, seed=240 + k))
    for k, (h, il) in enumerate(((35, 1), (49, 2), (63, 1), (67, 2), (81, 1), (95, 2), (3, 1), (17, 2), (31, 1), (2, 2))):
        cs.append(Case([FMT_422, FMT_444, FMT_4444][k % 3], 40, h, il, 3, 4, seed=250 + k))
    return cs


def option_cases():
    """quant_sel -1..4, bits_per_mb 128 / 8192, force_quant 1 / 7 / 64, alpha_bits 0 / 8 / 16, other vendor and colour bytes"""
    cs = []
    for k, qs in enumerate((-1, 0, 1, 2, 3, 4)):
        cs.append(Case([FMT_422, FMT_444, FMT_4444][k % 3], 72, 40, k % 3, k % 5, 4, quant_sel=qs, seed=300 + k))
    for k, bpm in enumerate((128, 8192)):
        cs.append(Case(FMT_422, 96, 48, 0, 2, 8, bits_per_mb=bpm, seed=310 + k))
        cs.append(Case(FMT_4444, 64, 32, 1, 4, 4, bits_per_mb=bpm, seed=315 + k))
    for k, fq in enumerate((1, 7, 64)):
        cs.append(Case([FMT_422, FMT_444, FMT_4444][k], 80, 36, k % 3, (k + 1) % 5, 8, force_quant=fq, seed=320 + k))
    for k, ab in enumerate((0, 8, 16)):
        cs.append(Case(FMT_4444, 56, 40, k % 3, 4, 2, alpha_bits=ab, alpha="runs", seed=330 + k))
    cs.append(Case(FMT_444, 48, 32, 0, 3, 4, vendor=b"ap\x7f\xff", colour=(1, 13, 9), seed=340))
    cs.append(Case(FMT_4444, 48, 32, 2, 1, 1, vendor=b"xyzw", colour=(255, 0, 128), seed=341))
    return cs


def content_cases():
    """content that takes every path: proxy with bits_per_mb 128 (past max_quant into q >= 16, and noise out at 128), flat frames,
    0 / 1023 extremes, alpha runs and noise at both depths, and the largest slices 10-bit samples give (0 / 1023 extremes at q = 1)"""
    cs = [
        Case(FMT_422, 96, 48, 0, 0, 8, bits_per_mb=128, content="noise", seed=400),
        Case(FMT_422, 96, 48, 0, 0, 8, bits_per_mb=128, content="natural", seed=400),
        Case(FMT_4444, 64, 32, 1, 0, 4, bits_per_mb=128, content="noise", alpha="noise", seed=401),
        Case(FMT_444, 64, 32, 0, 0, 8, bits_per_mb=128, content="extremes", seed=402),
        Case(FMT_422, 64, 48, 0, 2, 8, content="flat", seed=403),
        Case(FMT_4444, 48, 32, 2, 4, 4, content="flat", alpha="runs", seed=404),
        Case(FMT_422, 64, 32, 1, 3, 8, content="extremes", seed=405),
        Case(FMT_4444, 64, 32, 0, 4, 8, alpha_bits=8, alpha="noise", seed=406),
        Case(FMT_4444, 64, 32, 0, 4, 8, alpha_bits=16, alpha="runs", seed=407),
        Case(FMT_444, 128, 16, 0, 3, 8, content="extremes", seed=408),
        Case(FMT_4444, 128, 16, 0, 4, 8, content="extremes", alpha="noise", seed=409),
        Case(FMT_444, 128, 16, 0, 3, 8, content="extremes", force_quant=1, seed=410),
    ]
    return cs


def all_cases():
    return matrix_cases() + edge_cases() + option_cases() + content_cases()
