"""Pictures and macroblock records for the mpegvideo motion compensation tests (tests/test_mpv_mc_cpu.py, tests/test_gpu_mpv_mc.py), and the
four ways of running them: the reference's own ff_mpv_motion through oracle/_ref/libmpvmcref.so, its plain-C restatement
(oracle/port/orc_mpvmc.c), the product compiled for the host (tests/hostsim/mpv_mc_hostsim.cpp) and the product on the GPU.  Every plane buffer, its padding included, holds random bytes, so a kernel
that clamps where the reference reads directly, or writes outside its macroblock, gives a different buffer."""
import ctypes as C
import os
import subprocess

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
MPVMC_REF = os.path.join(ROOT, "oracle", "_ref", "libmpvmcref.so")
SIM_LIB = os.path.join(HERE, "hostsim", "libmpvmc_hostsim.so")

REC = np.dtype([("mb_x", "<u2"), ("mb_y", "<u2"), ("mv_dir", "u1"), ("mv_type", "u1"), ("field_select", "u1", (2, 2)),
                ("mv", "<i2", (2, 4, 2)), ("pad", "u1", (2,))])
assert REC.itemsize == 44
T16X16, T8X8, T16X8, TFIELD, TDMV = 0, 1, 2, 3, 4
TOP, BOTTOM, FRAME = 1, 2, 3
BUG_QPEL_CHROMA, BUG_QPEL_CHROMA2 = 64, 256
PRM = ("linesize", "uvlinesize", "pic_linesize", "pic_uvlinesize", "mb_width", "mb_height", "width", "height", "h_edge_pos", "v_edge_pos",
       "out_format", "picture_structure", "first_field", "b_picture", "no_rounding", "quarter_sample", "workaround_bugs")


class Picture:
    """One picture as an MpegEncContext would describe it, with host planes: `frame` is the frame being reconstructed (dest and cur),
    `last` / `next` the reference frames.  Each plane buffer has (16 * mb_height + 2) rows (chroma 8 * mb_height + 2) of `linesize` bytes."""

    def __init__(self, rng, fmt, mb_w, mb_h, structure=FRAME, first_field=1, b=0, no_rnd=0, qpel=0, bugs=0, width=None, height=None,
                 refs=None, custom_edges=False):
        self.p = dict(out_format=fmt, mb_width=mb_w, mb_height=mb_h, picture_structure=structure, first_field=first_field, b_picture=b,
                      no_rounding=no_rnd, quarter_sample=qpel, workaround_bugs=bugs)
        ls, uvls = 16 * mb_w + 32, 8 * mb_w + 24
        k = 1 if structure == FRAME else 2
        w = width if width is not None else 16 * mb_w
        h = height if height is not None else 16 * mb_h
        self.p.update(linesize=ls, uvlinesize=uvls, pic_linesize=k * ls, pic_uvlinesize=k * uvls, width=w, height=h)
        if fmt == 0:
            self.p.update(h_edge_pos=16 * mb_w, v_edge_pos=16 * mb_h if structure == FRAME else 8 * mb_h)
        elif custom_edges:
            # H.263 and H.263+ custom picture sizes: the edges stay at the macroblock grid (mpegvideo.c:634-635) while width / height
            # are smaller, so the av_clip to [-16, width] of a 4MV block and the dxy masking there are visible
            self.p.update(h_edge_pos=16 * mb_w, v_edge_pos=16 * mb_h)
        else:
            self.p.update(h_edge_pos=w, v_edge_pos=h)          # MPEG-4 (mpeg4videodec.c:2318-2319)
        self.frame = self.planes(rng)
        self.last, self.next = refs if refs is not None else (self.planes(rng), self.planes(rng))
        self.recs = np.zeros(0, REC)

    def planes(self, rng):
        mb_w, mb_h, ls, uvls = self.p["mb_width"], self.p["mb_height"], self.p["linesize"], self.p["uvlinesize"]
        return [rng.integers(0, 256, (16 * mb_h + 2, ls), dtype=np.uint8), rng.integers(0, 256, (8 * mb_h + 2, uvls), dtype=np.uint8),
                rng.integers(0, 256, (8 * mb_h + 2, uvls), dtype=np.uint8)]

    @property
    def dest_off(self):
        """current_picture.f->data of a bottom field starts one line down (mpegvideo.c:1224-1234)"""
        bottom = self.p["picture_structure"] == BOTTOM
        return [self.p["linesize"] if bottom else 0, self.p["uvlinesize"] if bottom else 0, self.p["uvlinesize"] if bottom else 0]

    @property
    def mb_rows(self):
        return self.p["mb_height"] if self.p["picture_structure"] == FRAME else self.p["mb_height"] // 2

    def accepted(self, recs=None):
        """the records ff_mpv_motion_batch_cuda takes (include/avdsp_b200.h): the rest leave their macroblock untouched"""
        r = self.recs if recs is None else recs
        frame, h263 = self.p["picture_structure"] == FRAME, self.p["out_format"] == 2
        ok = (r["mb_x"] < self.p["mb_width"]) & (r["mb_y"] < self.mb_rows) & (r["mv_dir"] <= 7) & (r["mv_type"] <= TDMV)
        t = r["mv_type"]
        if h263:
            ok &= (t == T16X16) | (t == T8X8)
        else:
            ok &= (t != T8X8) & ~(frame & (t == T16X8)) & ~((not frame) & (t == T16X16))
        return ok

    def prm(self):
        return np.array([self.p[k] for k in PRM], np.int32)


# ------------------------------------------------------------------------------------------------------------------------------- records

def mv_types(fmt, structure):
    if fmt == 2:
        return [T16X16, T8X8]
    return [T16X16, TFIELD, TDMV] if structure == FRAME else [TFIELD, T16X8, TDMV]


def _component(rng, kind, unit, base, edges, blk):
    """one vector component: small, far outside, or placing the block exactly at / one step inside / one step outside an edge (the
    picture edge, and the width / height where they differ from it)"""
    if kind == 0:
        return int(rng.integers(-6 * unit, 6 * unit + 1))
    if kind == 1:
        return int(np.clip(int(rng.choice([-32768, 32767, -20000, 20000, -4000, 4000])) + int(rng.integers(-3, 4)), -32768, 32767))
    edge = int(rng.choice(edges))
    t = int(rng.choice([-blk - 1, -blk, -blk + 1, -1, 0, 1, edge - blk - 1, edge - blk, edge - blk + 1, edge - 1, edge, edge + 1]))
    return int(np.clip(unit * (t - base) + int(rng.integers(0, unit)), -32768, 32767))


def make_records(rng, pic, n=None, far=0.1, edge=0.35, types=None):
    """one record per macroblock (a random subset, in random order) with vectors of every kind and every type the family has"""
    p = pic.p
    fmt, structure = p["out_format"], p["picture_structure"]
    mbs = [(x, y) for y in range(pic.mb_rows) for x in range(p["mb_width"])]
    rng.shuffle(mbs)
    mbs = mbs[:n] if n else mbs
    recs = np.zeros(len(mbs), REC)
    types = types or mv_types(fmt, structure)
    unit = 4 if (fmt == 2 and p["quarter_sample"]) else 2
    for i, (x, y) in enumerate(mbs):
        r = recs[i]
        r["mb_x"], r["mb_y"] = x, y
        r["mv_type"] = types[int(rng.integers(0, len(types)))]
        r["mv_dir"] = int(rng.choice([1, 2, 3, 3, 7])) if p["b_picture"] else int(rng.choice([1, 1, 1, 2, 3]))
        r["field_select"] = rng.integers(0, 2, (2, 2))
        field_rows = fmt == 0 and (structure != FRAME or r["mv_type"] in (TFIELD, TDMV))
        vh = p["v_edge_pos"] // (2 if (structure == FRAME and field_rows) else 1)
        yb = y * (8 if (structure == FRAME and field_rows) else 16)
        for d in range(2):
            for k in range(4):
                u = rng.random()
                kind = 1 if u < far else 2 if u < far + edge else 0
                sub_x, sub_y = (8 * (k & 1), 8 * (k >> 1)) if r["mv_type"] == T8X8 else (0, 0)
                blk = 8 if r["mv_type"] == T8X8 else 16
                r["mv"][d, k, 0] = _component(rng, kind, unit, 16 * x + sub_x, [p["h_edge_pos"], p["width"]], blk)
                r["mv"][d, k, 1] = _component(rng, kind if rng.random() < 0.7 else 0, unit, yb + sub_y,
                                              [vh] if fmt == 0 else [vh, p["height"]], blk)
    pic.recs = recs
    return recs


# ------------------------------------------------------------------------------------------------------------------------------- runners

def ref_lib():
    """the reference (ref_mpvmc_picture), or None where oracle/_ref was not built"""
    if not os.path.exists(MPVMC_REF):
        return None
    lib = C.CDLL(MPVMC_REF)
    lib.picture = lib.ref_mpvmc_picture
    lib.picture.restype = C.c_int
    lib.picture.argtypes = [C.c_void_p] * 5 + [C.c_void_p, C.c_size_t]
    lib.ref_mpvmc_impl.argtypes = [C.POINTER(C.c_void_p), C.POINTER(C.c_void_p)]
    return lib


class _Port:
    """the plain-C restatement (orc_mpvmc_picture in oracle/liboracle_port.so), called like the reference"""

    def __init__(self):
        from oracle import loader
        self.picture = loader.port().lib.orc_mpvmc_picture
        self.picture.restype = C.c_int
        self.picture.argtypes = [C.c_void_p] * 5 + [C.c_void_p, C.c_size_t]


def port_lib():
    return _Port()


def checker_lib():
    """the strongest checker available: the compiled reference where it was built, else the port (which the CPU suite pins to it)"""
    return ref_lib() or port_lib()


def _ptrs(planes, offs=(0, 0, 0)):
    return (C.c_void_p * 3)(*[a.ctypes.data + o for a, o in zip(planes, offs)])


def run_ref(lib, pic, frame=None):
    """the reference (or the port: anything from ref_lib / port_lib) over the picture's accepted records; returns the reconstructed
    frame planes (copies)"""
    f = [a.copy() for a in (frame or pic.frame)]
    recs = np.ascontiguousarray(pic.recs[pic.accepted()])
    prm = pic.prm()                      # held here: .ctypes.data alone does not keep the array alive during the call
    assert lib.picture(_ptrs(f, pic.dest_off), _ptrs(f), _ptrs(pic.last), _ptrs(pic.next), prm.ctypes.data,
                                 recs.ctypes.data, len(recs)) == 0
    return f


def sim_lib():
    """tests/hostsim/mpv_mc_hostsim.cpp built into its own library (under a temporary name, then renamed into place)"""
    hs = os.path.join(HERE, "hostsim")
    csrc = os.path.join(ROOT, "libav_b200", "csrc")
    src = os.path.join(hs, "mpv_mc_hostsim.cpp")
    deps = [src, os.path.join(hs, "shim", "cuda_runtime.h"), os.path.join(csrc, "mpv_mc.cu"), os.path.join(csrc, "mpv_mc_block.cuh"),
            os.path.join(csrc, "common.cuh"), os.path.join(ROOT, "include", "avdsp_b200.h")]
    if not os.path.exists(SIM_LIB) or any(os.path.getmtime(d) > os.path.getmtime(SIM_LIB) for d in deps):
        tmp = "%s.%d.tmp" % (SIM_LIB, os.getpid())
        subprocess.run(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-x", "c++", "-DAVB_HOSTSIM", "-I", os.path.join(hs, "shim"), "-I", csrc,
                        "-Wno-unknown-pragmas", "-Wl,--no-undefined", "-o", tmp, src], check=True)
        os.replace(tmp, SIM_LIB)
    lib = C.CDLL(SIM_LIB)
    lib.ff_mpv_motion_batch_cuda.restype = C.c_int
    lib.ff_mpv_motion_batch_cuda.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_void_p]
    lib.hostsim_last_error.restype = C.c_char_p
    return lib


def picture_struct(pic, dest, cur, last, nxt, recs_ptr, n_recs):
    """FFMpvMCPicture from plane base pointers (host or device addresses)"""
    from libav_b200 import tables
    s = tables.FFMpvMCPicture()
    for i in range(3):
        s.dest[i] = dest[i] + pic.dest_off[i]
        s.cur[i], s.last[i], s.next[i] = cur[i], last[i], nxt[i]
    for k in PRM:
        setattr(s, k, int(pic.p[k]))
    s.chroma_format = 1
    s.recs, s.n_recs = recs_ptr, n_recs
    return s


def run_sim(lib, pics):
    """the host-compiled product over all the pictures in one call; returns (frames, rejected count)"""
    frames = [[a.copy() for a in pic.frame] for pic in pics]
    recs = [np.ascontiguousarray(pic.recs) for pic in pics]
    arr = (type(picture_struct(pics[0], [0] * 3, [0] * 3, [0] * 3, [0] * 3, None, 0)) * len(pics))()
    for i, pic in enumerate(pics):
        base = [a.ctypes.data for a in frames[i]]
        arr[i] = picture_struct(pic, base, base, [a.ctypes.data for a in pic.last], [a.ctypes.data for a in pic.next], recs[i].ctypes.data, len(recs[i]))
    rej = np.zeros(1, np.uint32)
    rc = lib.ff_mpv_motion_batch_cuda(C.cast(arr, C.c_void_p), len(pics), rej.ctypes.data, None)
    assert rc == 0, lib.hostsim_last_error()
    return frames, int(rej[0])


class GpuPictures:
    """the pictures' planes and records in device memory, and the FFMpvMCPicture array that describes them"""

    def __init__(self, pics):
        from libav_b200 import device, tables
        dev = lambda a: device.DevBuf.from_numpy(np.ascontiguousarray(a))
        self.pics = pics
        self.keep, self.frames, self.arr = [], [], (tables.FFMpvMCPicture * len(pics))()
        ref_bufs = {}
        for i, pic in enumerate(pics):
            fr = [dev(a) for a in pic.frame]
            refs = []
            for planes in (pic.last, pic.next):
                key = id(planes)
                if key not in ref_bufs:
                    ref_bufs[key] = [dev(a) for a in planes]
                refs.append(ref_bufs[key])
            rb = dev(pic.recs) if len(pic.recs) else None
            self.keep += [rb]
            self.frames.append(fr)
            base = [b.ptr for b in fr]
            self.arr[i] = picture_struct(pic, base, base, [b.ptr for b in refs[0]], [b.ptr for b in refs[1]], rb.ptr if rb else None, len(pic.recs))
        self.keep.append(ref_bufs)
        self.rej = device.DevBuf.from_numpy(np.zeros(1, np.uint32))

    def download(self):
        return [[b.download(np.uint8, a.shape) for b, a in zip(fr, pic.frame)] for fr, pic in zip(self.frames, self.pics)]

    def rejected(self):
        return int(self.rej.download(np.uint32, (1,))[0])


def first_diff(got, want):
    for pl in range(3):
        if not np.array_equal(got[pl], want[pl]):
            yx = np.argwhere(got[pl] != want[pl])[0]
            return "plane %d first difference at row %d col %d: %d vs %d" % (pl, yx[0], yx[1], got[pl][tuple(yx)], want[pl][tuple(yx)])
    return None


# ------------------------------------------------------------------------------------------------------------------------------- residual

def residual_batch(checker, pics, pi, pl, tr, dq, mode, offs, stride, clear, seed, alt=0, aic=0):
    """one residual batch of ff_mpv_flush_pictures_cuda on plane `pl` of picture `pi`: blocks at byte offsets `offs` of the plane buffer
    (so a bottom field's line offset is inside them), coefficients (and dequantiser records / tables for dq >= 0) from test_gpu_mpv.make_case"""
    from test_gpu_mpv import make_case
    n = len(offs)
    blocks, rec, t, intra, inter = make_case(checker, dq if dq >= 0 else 1, n, seed, alt, aic, wild=False)
    return dict(pi=pi, pl=pl, tr=tr, dq=dq, mode=mode, off=np.asarray(offs, np.uint32), stride=stride, clear=clear, blocks=blocks, rec=rec,
                t=t, intra=intra, inter=inter, alt=alt, aic=aic)


def xvid_checker():
    """the Xvid IDCT checker: the compiled reference where it was built, else the port"""
    from test_xvid_idct import XVID_REF, Xvid
    from oracle import loader
    return Xvid(C.CDLL(XVID_REF), "ref_") if os.path.exists(XVID_REF) else Xvid(loader.port().lib, "orc_")


def apply_residual(checker, xv, frames, batches):
    """the chained checker's residual half, on host frames in place, batch after batch: dequantise (inter kinds skip blocks with
    last_index < 0), then idct_put / idct_add through the simple or the Xvid IDCT oracle.  Returns, per batch, the mask of the blocks the
    call consumes (what `clear` zeroes)."""
    from test_gpu_mpv import INTER, oracle_dequant
    from oracle import loader
    keeps = []
    for b in batches:
        f, n = frames[b["pi"]][b["pl"]], len(b["off"])
        if b["dq"] >= 0:
            deq = oracle_dequant(checker, b["dq"], b["blocks"], b["rec"], b["intra"], b["inter"], b["alt"], b["aic"])
            m = 1 if b["dq"] in INTER else 0
            keep = np.ones(n, bool) if m == 0 else b["rec"]["last"] >= 0
        else:
            deq, m, keep = b["blocks"], b["mode"], np.ones(n, bool)
        idx = np.flatnonzero(keep)
        sub, suboff = np.ascontiguousarray(deq[idx]), np.ascontiguousarray(b["off"][idx])
        if b["tr"] == 0:
            checker.idct_batch(m, loader.ptr(sub), loader.ptr(f), loader.ptr(suboff), b["stride"], len(idx), 1)
        else:
            f[...] = xv.batch(m, sub, f, suboff, b["stride"])[1]
        keeps.append(keep)
    return keeps


class GpuResidual:
    """the batches in device memory as an FFMpvResidualBatch array addressing the planes of `g` (a GpuPictures)"""

    def __init__(self, g, batches):
        from libav_b200 import device, tables
        self.keep, items = [], []
        for b in batches:
            d_b, d_o = device.DevBuf.from_numpy(np.ascontiguousarray(b["blocks"])), device.DevBuf.from_numpy(b["off"])
            d_r = device.DevBuf.from_numpy(np.ascontiguousarray(b["rec"])) if b["dq"] >= 0 else None
            x = tables.FFMpvResidualBatch()
            x.transform, x.dequant, x.mode, x.clear = b["tr"], b["dq"], b["mode"], b["clear"]
            x.tables = C.cast(C.pointer(b["t"]), C.c_void_p) if b["dq"] >= 0 else None
            x.recs = d_r.ptr if d_r else None
            x.blocks, x.frame, x.dst_off, x.stride, x.n = d_b.ptr, g.frames[b["pi"]][b["pl"]].ptr, d_o.ptr, b["stride"], len(b["off"])
            self.keep += [d_b, d_o, d_r, b["t"]]
            items.append(x)
        self.blocks = [self.keep[4 * i] for i in range(len(batches))]
        self.arr = (tables.FFMpvResidualBatch * len(items))(*items)

    def work(self, g):
        from libav_b200 import tables
        w = tables.FFMpvPictureWork()
        w.pictures, w.n_pictures, w.rejected = C.cast(g.arr, C.c_void_p), len(g.pics), g.rej.ptr
        w.residual, w.n_residual = C.cast(self.arr, C.c_void_p), len(self.arr)
        return w


def decoder_residual(checker, pics, rng, intra_share=0.08, coded=0.5, xvid=False, clear=1):
    """the residual a decoder would record for these pictures: a share of the macroblocks turned intra (their MC records dropped, all six
    blocks coded), the inter macroblocks with each block coded at probability `coded`; in frame pictures half of the macroblocks use field
    DCT (luma stride 2 * linesize, lower blocks one line down).  MPEG-1 / 2: the levels are dequantised while parsing, so intra blocks are
    idct_put and inter blocks idct_add through the simple IDCT.  H.263 / MPEG-4 (Xvid-written when `xvid`): intra blocks are put_dct with
    the h263_intra kind (5) fused, inter blocks add_dct.  One batch per picture, plane and (intra / inter, frame / field DCT)."""
    batches = []
    for pi, pic in enumerate(pics):
        keep = rng.random(len(pic.recs)) >= intra_share
        intra_mbs = {(int(r["mb_x"]), int(r["mb_y"])) for r in pic.recs[~keep]}
        pic.recs = pic.recs[keep]
        inter_mbs = [(int(r["mb_x"]), int(r["mb_y"])) for r in pic.recs]
        frame = pic.p["picture_structure"] == FRAME
        ls, uvls, pls, puvls = pic.p["linesize"], pic.p["uvlinesize"], pic.p["pic_linesize"], pic.p["pic_uvlinesize"]
        d0 = pic.dest_off
        groups = {}
        for intra, mbs in ((1, sorted(intra_mbs)), (0, inter_mbs)):
            for (x, y) in mbs:
                fd = frame and pic.p["out_format"] == 0 and rng.random() < 0.5
                o = d0[0] + 16 * y * pls + 16 * x
                lower = ls if fd else 8 * pls
                for k, bo in enumerate((o, o + 8, o + lower, o + lower + 8)):
                    if intra or rng.random() < coded:
                        groups.setdefault((intra, 0, fd), []).append(bo)
                for p in (1, 2):
                    if intra or rng.random() < coded:
                        groups.setdefault((intra, p, False), []).append(d0[p] + 8 * y * puvls + 8 * x)
        for (intra, pl, fd), offs in sorted(groups.items()):
            stride = (2 * ls if fd else pls) if pl == 0 else puvls
            if pic.p["out_format"] == 2:
                tr, dq, mode = (1 if xvid else 0), (5 if intra else -1), (0 if intra else 1)
            else:
                tr, dq, mode = 0, -1, (0 if intra else 1)
            batches.append(residual_batch(checker, pics, pi, pl, tr, dq, mode, offs, stride, clear, int(rng.integers(1 << 30))))
    return batches
