"""Pictures, records and runners for the MPEG-2 4:2:2 / 4:4:4 and interlaced MPEG-4 motion compensation tests (tests/test_mpv_ilace_cpu.py,
tests/test_gpu_mpv_ilace.py), on top of tests/mpv_mc_cases.py and tests/mpv_gmc_cases.py, whose behaviour they leave as it is.

  CfPicture     an MPEG-2 picture in chroma format 1, 2 or 3: chroma planes (16 >> chroma_x_shift) * mb_width wide (plus padding) and
                (16 >> chroma_y_shift) * mb_height rows (plus two), random bytes everywhere
  IlacePicture  an MPEG-4 frame picture with interlaced set: FIELD records are taken besides 16X16 and 8X8 (and an S-VOP when .sprite is
                set, as in mpv_gmc_cases)

The checker is the reference's own ff_mpv_motion: ref_mpvmc_cf_picture (oracle/_ref/libmpvcfref.so) for the chroma formats,
ref_mpvmc_picture / ref_mpvmc_gmc_picture for interlaced MPEG-4, which need no glue of their own (the real function runs FIELD records of
FMT_H263 pictures)."""
import ctypes as C

import numpy as np

from oracle import loader

import mpv_gmc_cases as G
import mpv_mc_cases as M

BUG_HPEL_CHROMA = 2048


class CfPicture(M.Picture):
    """an MPEG-2 picture (out_format 0) in chroma format `cf`"""

    def __init__(self, rng, cf, mb_w, mb_h, **kw):
        self.cf, self.interlaced = cf, 0
        super().__init__(rng, 0, mb_w, mb_h, **kw)

    @property
    def shifts(self):
        return int(self.cf != 3), int(self.cf == 1)

    def planes(self, rng):
        cx, cy = self.shifts
        mb_w, mb_h, ls = self.p["mb_width"], self.p["mb_height"], self.p["linesize"]
        uvls = (16 >> cx) * mb_w + 24
        k = 1 if self.p["picture_structure"] == M.FRAME else 2
        self.p.update(uvlinesize=uvls, pic_uvlinesize=k * uvls)
        ch = (16 >> cy) * mb_h + 2
        return [rng.integers(0, 256, (16 * mb_h + 2, ls), dtype=np.uint8), rng.integers(0, 256, (ch, uvls), dtype=np.uint8),
                rng.integers(0, 256, (ch, uvls), dtype=np.uint8)]


class IlacePicture(M.Picture):
    """an MPEG-4 frame picture (out_format 2) of an interlaced VOL"""

    def __init__(self, rng, mb_w, mb_h, **kw):
        self.cf, self.interlaced = 1, 1
        super().__init__(rng, 2, mb_w, mb_h, **kw)

    def accepted(self, recs=None):
        r = self.recs if recs is None else recs
        t = r["mv_type"]
        ok = (r["mb_x"] < self.p["mb_width"]) & (r["mb_y"] < self.mb_rows) & (r["mv_dir"] <= 7)
        return ok & ((t == M.T16X16) | (t == M.T8X8) | (t == M.TFIELD))


def ilace_records(rng, pic, field=0.5, far=0.1, edge=0.35, mcsel=0.0, direct=0.2):
    """records of an interlaced MPEG-4 picture: 16X16 / 8X8 as tests/mpv_mc_cases.py makes them, a share `field` turned FIELD with
    vectors of every kind in field rows (blocks exactly at / one step inside / outside the top and bottom edges of the field, which the
    reference emulates in frame rows), random field_select pairs; in a B picture a share `direct` of the FIELD records as B-direct makes
    them (mv_dir 7, field_select[1] = {0, 1}).  S-VOPs: mcsel on a share of the 16X16 records.  The G.REC layout (mcsel at byte 42)."""
    p = pic.p
    old = M.make_records(rng, pic, far=far, edge=edge, types=[M.T16X16, M.T8X8])
    recs = np.zeros(len(old), G.REC)
    for name in M.REC.names:
        if name != "pad":
            recs[name] = old[name]
    unit = 4 if p["quarter_sample"] else 2
    vh = p["v_edge_pos"] // 2
    for r in recs:
        if rng.random() >= field:
            continue
        r["mv_type"] = M.TFIELD
        x, y = int(r["mb_x"]), int(r["mb_y"])
        for d in range(2):
            for i in range(2):
                u = rng.random()
                kind = 1 if u < far else 2 if u < far + edge else 0
                r["mv"][d, i, 0] = M._component(rng, kind, unit, 16 * x, [p["h_edge_pos"], p["width"]], 16)
                r["mv"][d, i, 1] = M._component(rng, kind if rng.random() < 0.8 else 0, unit, 8 * y, [vh, p["height"] // 2], 8)
        if p["b_picture"] and rng.random() < direct:
            r["mv_dir"] = 7
            r["field_select"][1] = (0, 1)
    if mcsel:
        recs["mcsel"] = (recs["mv_type"] == M.T16X16) & (rng.random(len(recs)) < mcsel)
    pic.recs = recs
    return recs


def ilace_picture(rng, mb_w, mb_h, b=0, qpel=0, bugs=0, no_rnd=0, ragged=False, sprite=False, **kw):
    """an interlaced MPEG-4 picture with records; `ragged`: width / height not a multiple of 16; `sprite`: an S-VOP (P-like, random
    sprite trajectory, mcsel on 16X16 records)"""
    size = dict(width=16 * mb_w - int(rng.integers(1, 15)), height=16 * mb_h - 2 * int(rng.integers(1, 7))) if ragged else {}
    pic = IlacePicture(rng, mb_w, mb_h, b=b, qpel=qpel, bugs=bugs, no_rnd=no_rnd, **size)
    ilace_records(rng, pic, mcsel=0.5 if sprite else 0.0, **kw)
    if sprite:
        q = pic.p
        pic.sprite = G.random_params(rng, q["width"], q["height"], mb_w, mb_h, q["h_edge_pos"], q["v_edge_pos"])
    return pic


def cf_picture(rng, cf, mb_w, mb_h, structure=M.FRAME, first_field=1, b=0, no_rnd=0, refs=None, **kw):
    pic = CfPicture(rng, cf, mb_w, mb_h, structure=structure, first_field=first_field, b=b, no_rnd=no_rnd, refs=refs)
    M.make_records(rng, pic, **kw)
    return pic


# ------------------------------------------------------------------------------------------------------------------------------- runners

def cf_ref_lib():
    """ref_mpvmc_cf_picture, or None where oracle/_ref was not built"""
    lib = loader.ref_lib("mpvcf")
    if lib is None:
        return None
    lib.cf_picture = lib.ref_mpvmc_cf_picture
    lib.cf_picture.restype = C.c_int
    lib.cf_picture.argtypes = [C.c_void_p] * 5 + [C.c_void_p, C.c_size_t, C.c_int]
    return lib


def have_reference():
    return cf_ref_lib() is not None and M.ref_lib() is not None and G.ref_lib() is not None


def run_ref(pic):
    """the reference over the picture's accepted records; returns the reconstructed frame planes (copies)"""
    if getattr(pic, "sprite", None) is not None:
        return G.run_ref(G.ref_lib(), pic)
    if pic.cf == 1:
        return M.run_ref(M.ref_lib(), pic)
    f = [a.copy() for a in pic.frame]
    recs, prm = np.ascontiguousarray(pic.recs[pic.accepted()]), pic.prm()
    assert cf_ref_lib().cf_picture(M._ptrs(f, pic.dest_off), M._ptrs(f), M._ptrs(pic.last), M._ptrs(pic.next), prm.ctypes.data,
                                   recs.ctypes.data, len(recs), pic.cf) == 0
    return f


def set_fields(s, pic):
    """chroma_format, interlaced and the sprite fields of an FFMpvMCPicture from the picture"""
    s.chroma_format = getattr(pic, "cf", 1)
    s.interlaced = getattr(pic, "interlaced", 0)
    return G.set_sprite(s, pic)


def run_sim(lib, pics):
    """the host-compiled product over all the pictures in one call; returns (frames, rejected count)"""
    from libav_b200 import tables
    frames = [[a.copy() for a in pic.frame] for pic in pics]
    recs = [np.ascontiguousarray(pic.recs) for pic in pics]
    arr = (tables.FFMpvMCPicture * len(pics))()
    for i, pic in enumerate(pics):
        base = [a.ctypes.data for a in frames[i]]
        arr[i] = set_fields(M.picture_struct(pic, base, base, [a.ctypes.data for a in pic.last], [a.ctypes.data for a in pic.next],
                                             recs[i].ctypes.data, len(recs[i])), pic)
    rej = np.zeros(1, np.uint32)
    rc = lib.ff_mpv_motion_batch_cuda(C.cast(arr, C.c_void_p), len(pics), rej.ctypes.data, None)
    assert rc == 0, lib.avb200_last_error()
    return frames, int(rej[0])


class GpuPics(M.GpuPictures):
    """GpuPictures with each picture's chroma format, interlaced flag and sprite fields"""

    def __init__(self, pics):
        super().__init__(pics)
        for i, p in enumerate(pics):
            set_fields(self.arr[i], p)


# ------------------------------------------------------------------------------------------------------------------------------- residual

def residual(checker, pics, rng, xvid=False, intra_share=0.08, coded=0.5, clear=1):
    """M.decoder_residual for any chroma format and for interlaced MPEG-4: a share of the macroblocks turned intra (their records
    dropped), the blocks of inter macroblocks coded at probability `coded`.  Field DCT (interlaced_dct) in half the macroblocks of MPEG-2
    frame pictures and of interlaced MPEG-4 pictures: luma stride 2 * linesize, lower blocks one line down; in 4:2:2 / 4:4:4 the chroma
    blocks follow it (dct_linesize = uvlinesize << interlaced_dct, mpegvideo.c:1620-1635), so a chroma plane has 2 (4:2:2) or 4 (4:4:4)
    blocks per macroblock.  One batch per picture, plane and (intra / inter, frame / field DCT)."""
    batches = []
    for pi, pic in enumerate(pics):
        keep = rng.random(len(pic.recs)) >= intra_share
        intra_mbs = {(int(r["mb_x"]), int(r["mb_y"])) for r in pic.recs[~keep]}
        pic.recs = pic.recs[keep]
        inter_mbs = [(int(r["mb_x"]), int(r["mb_y"])) for r in pic.recs]
        frame = pic.p["picture_structure"] == M.FRAME
        h263 = pic.p["out_format"] == 2
        cf = getattr(pic, "cf", 1)
        cw, chh = 16 >> int(cf != 3), 16 >> int(cf == 1)
        ls, uvls, pls, puvls = pic.p["linesize"], pic.p["uvlinesize"], pic.p["pic_linesize"], pic.p["pic_uvlinesize"]
        d0 = pic.dest_off
        may_fd = frame and (not h263 or getattr(pic, "interlaced", 0))
        groups = {}
        for intra, mbs in ((1, sorted(intra_mbs)), (0, inter_mbs)):
            for (x, y) in mbs:
                fd = bool(may_fd and rng.random() < 0.5)
                o = d0[0] + 16 * y * pls + 16 * x
                lower = ls if fd else 8 * pls
                for bo in (o, o + 8, o + lower, o + lower + 8):
                    if intra or rng.random() < coded:
                        groups.setdefault((intra, 0, fd), []).append(bo)
                cfd = fd and cf != 1
                clower = uvls if cfd else 8 * puvls
                for p in (1, 2):
                    oc = d0[p] + chh * y * puvls + cw * x
                    blocks = [oc + dx + dy for dy in ((0, clower) if chh == 16 else (0,)) for dx in range(0, cw, 8)]
                    for bo in blocks:
                        if intra or rng.random() < coded:
                            groups.setdefault((intra, p, cfd), []).append(bo)
        for (intra, pl, fd), offs in sorted(groups.items()):
            stride = (2 * (ls if pl == 0 else uvls)) if fd else (pls if pl == 0 else puvls)
            if h263:
                tr, dq, mode = (1 if xvid else 0), (5 if intra else -1), (0 if intra else 1)
            else:
                tr, dq, mode = 0, -1, (0 if intra else 1)
            batches.append(M.residual_batch(checker, pics, pi, pl, tr, dq, mode, offs, stride, clear, int(rng.integers(1 << 30))))
    return batches
