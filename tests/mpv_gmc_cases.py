"""MPEG-4 S-VOPs for the global motion compensation tests (tests/test_mpv_gmc_cpu.py, tests/test_gpu_mpv_gmc.py): pictures of
tests/mpv_mc_cases.py whose records carry mcsel, their sprite parameters, and the ways of running them -- the reference's ff_mpv_motion on
S-VOPs (ref_mpvmc_gmc_picture in oracle/_ref/libmpvgmcref.so), its plain-C restatement (oracle/port/orc_mpvgmc.c), the product compiled for
the host (tests/hostsim/mpv_mc_hostsim.cpp) and the product on the GPU.

Sprite parameters come mostly from `trajectory`, a restatement of mpeg4_decode_sprite_trajectory (libavcodec/mpeg4videodec.c:168-385) for
a rectangular VOP: picture size, sprite_warping_accuracy 0..3, 0..3 warping points with their displacements, and the DivX 5.00 build 413
variant; a warp that is a translation is reduced to one point as the decoder reduces it.  `raw_params` adds sets no trajectory gives
readily: positions outside the picture on every side (all four clamp branches of ff_gmc_c, arithmetic shifts of negative positions,
blocks wholly outside), gmc1 offsets clipped to src_x == width / src_y == height, and whole / half-sample gmc1 offsets.

Domain: only parameters for which the reference's C is defined are generated -- 16 - sprite_shift[1] >= 0 (the chroma shift, the larger
one), and every intermediate of the trajectory, of gmc_motion's offsets and of ff_gmc_c's running sums fits int32 (checked in int64 over
every macroblock of the picture).  At accuracy 3 this bounds positions to about +-2048 samples, which 1920 x 1088 pictures still meet."""
import ctypes as C

import numpy as np

from oracle import loader
import mpv_mc_cases as M

REC = np.dtype([("mb_x", "<u2"), ("mb_y", "<u2"), ("mv_dir", "u1"), ("mv_type", "u1"), ("field_select", "u1", (2, 2)),
                ("mv", "<i2", (2, 4, 2)), ("mcsel", "u1"), ("pad", "u1")])
assert REC.itemsize == 44 and REC.fields["mcsel"][1] == 42
I32 = (-(1 << 31), (1 << 31) - 1)


def _fits(*vals):
    return all(I32[0] <= int(v) <= I32[1] for v in vals)


def _cdiv(a, b):
    """C integer division (truncation toward zero)"""
    q = abs(a) // abs(b)
    return q if (a >= 0) == (b > 0) else -q


def _rounded_div(a, b):
    return _cdiv(a + (b >> 1) if a >= 0 else a - (b >> 1), b)


def trajectory(w, h, acc, n_pts, d, divx413=False):
    """mpeg4_decode_sprite_trajectory's arithmetic for a w x h VOP and displacements d (n_pts x 2): (accuracy, real_sprite_warping_points,
    sprite_offset, sprite_delta), or None where an intermediate leaves int32 or the shift is negative (the C code is undefined there)"""
    a, rho = 2 << acc, 3 - acc
    r = 16 // a
    vop = [(0, 0), (w, 0), (0, h), (w, h)]
    dd = [[0, 0] for _ in range(4)]
    for i in range(n_pts):
        dd[i] = [int(d[i][0]), int(d[i][1])]
    alpha = beta = 0
    while (1 << alpha) < w:
        alpha += 1
    while (1 << beta) < h:
        beta += 1
    w2, h2 = 1 << alpha, 1 << beta
    sref = [[0, 0] for _ in range(3)]
    for k in range(2):
        if divx413:
            sref[0][k] = a * vop[0][k] + dd[0][k]
            sref[1][k] = a * vop[1][k] + dd[0][k] + dd[1][k]
            sref[2][k] = a * vop[2][k] + dd[0][k] + dd[2][k]
        else:
            sref[0][k] = (a >> 1) * (2 * vop[0][k] + dd[0][k])
            sref[1][k] = (a >> 1) * (2 * vop[1][k] + dd[0][k] + dd[1][k])
            sref[2][k] = (a >> 1) * (2 * vop[2][k] + dd[0][k] + dd[2][k])
    vr = [[0, 0], [0, 0]]
    vr[0][0] = 16 * (vop[0][0] + w2) + _rounded_div((w - w2) * (r * sref[0][0] - 16 * vop[0][0]) + w2 * (r * sref[1][0] - 16 * vop[1][0]), w)
    vr[0][1] = 16 * vop[0][1] + _rounded_div((w - w2) * (r * sref[0][1] - 16 * vop[0][1]) + w2 * (r * sref[1][1] - 16 * vop[1][1]), w)
    vr[1][0] = 16 * vop[0][0] + _rounded_div((h - h2) * (r * sref[0][0] - 16 * vop[0][0]) + h2 * (r * sref[2][0] - 16 * vop[2][0]), h)
    vr[1][1] = 16 * (vop[0][1] + h2) + _rounded_div((h - h2) * (r * sref[0][1] - 16 * vop[0][1]) + h2 * (r * sref[2][1] - 16 * vop[2][1]), h)
    inter = [x for row in sref + vr for x in row]
    if n_pts in (0, 1):
        if n_pts == 0:
            off = [[0, 0], [0, 0]]
        else:
            off = [[sref[0][0] - a * vop[0][0], sref[0][1] - a * vop[0][1]],
                   [((sref[0][0] >> 1) | (sref[0][0] & 1)) - a * (vop[0][0] // 2), ((sref[0][1] >> 1) | (sref[0][1] & 1)) - a * (vop[0][1] // 2)]]
        delta, shift = [[a, 0], [0, a]], [0, 0]
    elif n_pts == 2:
        s0, s1 = sref[0]
        off = [[(s0 << (alpha + rho)) + (-r * s0 + vr[0][0]) * (-vop[0][0]) + (r * s1 - vr[0][1]) * (-vop[0][1]) + (1 << (alpha + rho - 1)),
                (s1 << (alpha + rho)) + (-r * s1 + vr[0][1]) * (-vop[0][0]) + (-r * s0 + vr[0][0]) * (-vop[0][1]) + (1 << (alpha + rho - 1))],
               [(-r * s0 + vr[0][0]) * (-2 * vop[0][0] + 1) + (r * s1 - vr[0][1]) * (-2 * vop[0][1] + 1) + 2 * w2 * r * s0 - 16 * w2 + (1 << (alpha + rho + 1)),
                (-r * s1 + vr[0][1]) * (-2 * vop[0][0] + 1) + (-r * s0 + vr[0][0]) * (-2 * vop[0][1] + 1) + 2 * w2 * r * s1 - 16 * w2 + (1 << (alpha + rho + 1))]]
        delta = [[-r * s0 + vr[0][0], r * s1 - vr[0][1]], [-r * s1 + vr[0][1], -r * s0 + vr[0][0]]]
        shift = [alpha + rho, alpha + rho + 2]
        inter += [s0 << (alpha + rho), s1 << (alpha + rho), 2 * w2 * r * s0, 2 * w2 * r * s1]
    else:
        s0, s1 = sref[0]
        m = min(alpha, beta)
        w3, h3 = w2 >> m, h2 >> m
        e = alpha + beta + rho - m
        off = [[(s0 << e) + (-r * s0 + vr[0][0]) * h3 * (-vop[0][0]) + (-r * s0 + vr[1][0]) * w3 * (-vop[0][1]) + (1 << (e - 1)),
                (s1 << e) + (-r * s1 + vr[0][1]) * h3 * (-vop[0][0]) + (-r * s1 + vr[1][1]) * w3 * (-vop[0][1]) + (1 << (e - 1))],
               [(-r * s0 + vr[0][0]) * h3 * (-2 * vop[0][0] + 1) + (-r * s0 + vr[1][0]) * w3 * (-2 * vop[0][1] + 1) + 2 * w2 * h3 * r * s0 - 16 * w2 * h3 + (1 << (e + 1)),
                (-r * s1 + vr[0][1]) * h3 * (-2 * vop[0][0] + 1) + (-r * s1 + vr[1][1]) * w3 * (-2 * vop[0][1] + 1) + 2 * w2 * h3 * r * s1 - 16 * w2 * h3 + (1 << (e + 1))]]
        delta = [[(-r * s0 + vr[0][0]) * h3, (-r * s0 + vr[1][0]) * w3], [(-r * s1 + vr[0][1]) * h3, (-r * s1 + vr[1][1]) * w3]]
        shift = [e, e + 2]
        inter += [s0 << e, s1 << e, 2 * w2 * h3 * r * s0, 2 * w2 * h3 * r * s1]
    inter += [x for row in off + delta for x in row]
    if not _fits(*inter):
        return None
    if delta == [[a << shift[0], 0], [0, a << shift[0]]]:
        off = [[off[0][0] >> shift[0], off[0][1] >> shift[0]], [off[1][0] >> shift[1], off[1][1] >> shift[1]]]
        return acc, 1, off, [[a, 0], [0, a]]
    sy, sc = 16 - shift[0], 16 - shift[1]
    if sc < 0:
        return None
    off = [[v << sy for v in off[0]], [v << sc for v in off[1]]]
    delta = [[v << sy for v in delta[0]], [v << sy for v in delta[1]]]
    if not _fits(*[x for row in off + delta for x in row]):
        return None
    return acc, max(n_pts, 1), off, delta


def in_domain(params, mb_w, mb_h, h_edge, v_edge):
    """every intermediate of gmc_motion and ff_gmc_c fits int32 over the picture's macroblocks (trivially true for one point)"""
    acc, pts, off, d = params
    if pts == 1:
        return _fits(off[0][0] << (3 - acc), off[0][1] << (3 - acc), off[1][0] << (3 - acc), off[1][1] << (3 - acc))
    x = np.arange(mb_w, dtype=np.int64)[None, :]
    y = np.arange(mb_h, dtype=np.int64)[:, None]
    for c, bs in ((0, 16), (1, 8)):
        terms = [d[0][0] * x * bs, d[0][1] * y * bs, d[1][0] * x * bs, d[1][1] * y * bs]
        ox = off[c][0] + terms[0] + terms[1]
        oy = off[c][1] + terms[2] + terms[3]
        vals = terms + [off[c][0] + terms[0], off[c][1] + terms[2], ox, oy]
        # the running sums reach ox + dxx * 0..bs + dxy * 0..bs (the increments after the last column / row included)
        for cx in (0, bs):
            for cy in (0, bs):
                vals += [ox + d[0][0] * cx + d[0][1] * cy, oy + d[1][0] * cx + d[1][1] * cy]
        if not all(v.min() >= I32[0] and v.max() <= I32[1] for v in vals):
            return False
    return True


def random_params(rng, w, h, mb_w, mb_h, h_edge, v_edge, pts=None, acc=None, scale=None):
    """sprite parameters from a random trajectory inside the domain"""
    for _ in range(200):
        a = int(rng.integers(0, 4)) if acc is None else acc
        n = int(rng.integers(0, 4)) if pts is None else pts
        sc = scale if scale is not None else int(rng.choice([4, 16, 64, 256]))
        d = rng.integers(-sc, sc + 1, (3, 2))
        p = trajectory(w, h, a, n, d, divx413=bool(rng.random() < 0.25))
        if p is not None and in_domain(p, mb_w, mb_h, h_edge, v_edge):
            return p
    raise AssertionError("no trajectory inside the domain")


def raw_params(rng, pic, kind, acc, no_rnd=0):
    """hand-set parameters (see the module doc): kind 'clamp' (positions on every side of the picture, also wholly outside), 'edge1'
    (gmc1 clipped to width / height), 'hpel1' (gmc1 whole / half-sample offsets)"""
    p = pic.p
    W, H = p["width"], p["height"]
    if kind == "clamp":
        s = 16 + acc + 1
        for _ in range(200):
            px, py = int(rng.integers(-3 * 16, W + 3 * 16)), int(rng.integers(-3 * 16, H + 3 * 16))
            zoom = [[int((1 << s) * (1 + rng.uniform(-0.6, 0.6))), int((1 << s) * rng.uniform(-0.5, 0.5))],
                    [int((1 << s) * rng.uniform(-0.5, 0.5)), int((1 << s) * (1 + rng.uniform(-0.6, 0.6)))]]
            off = [[(px << s) + int(rng.integers(0, 1 << s)), (py << s) + int(rng.integers(0, 1 << s))],
                   [((px >> 1) << s) + int(rng.integers(0, 1 << s)), ((py >> 1) << s) + int(rng.integers(0, 1 << s))]]
            prm = (acc, int(rng.integers(2, 4)), off, zoom)
            if _fits(*[x for row in off + zoom for x in row]) and in_domain(prm, p["mb_width"], p["mb_height"], p["h_edge_pos"], p["v_edge_pos"]):
                return prm
        raise AssertionError("no raw parameters inside the domain")
    g = 2 << acc
    if kind == "edge1":
        ox = (W + int(rng.integers(0, 40))) * g + int(rng.integers(0, g)) if rng.random() < 0.5 else int(rng.integers(-40 * g, 40 * g))
        oy = (H + int(rng.integers(0, 40))) * g + int(rng.integers(0, g)) if rng.random() < 0.5 else int(rng.integers(-40 * g, 40 * g))
        off = [[ox, oy], [ox // 2 + int(rng.integers(0, 2)), oy // 2 + int(rng.integers(0, 2))]]
    else:
        step = 1 << acc                                      # (v << (3 - acc)) & 7 == 0: a whole or half luma sample
        off = [[int(rng.integers(-30, 30)) * step, int(rng.integers(-30, 30)) * step],
               [int(rng.integers(-60, 60)), int(rng.integers(-60, 60))]]
    return acc, 1, off, [[g, 0], [0, g]]


def svop(rng, mb_w, mb_h, params=None, no_rnd=0, qpel=0, ragged=False, mcsel=0.7, intra=0.08, types=(M.T16X16, M.T8X8), far=0.1, edge=0.35):
    """an MPEG-4 S-VOP: records of every kind of tests/mpv_mc_cases.py (16X16 and 8X8, half- or quarter-sample) with mcsel set on a
    share `mcsel` of them (8X8 ones included: ignored there, as in the C code), a share `intra` of the macroblocks without a record"""
    kw = dict(width=16 * mb_w - int(rng.integers(1, 15)), height=16 * mb_h - int(rng.integers(1, 15))) if ragged else {}
    pic = M.Picture(rng, 2, mb_w, mb_h, no_rnd=no_rnd, qpel=qpel, **kw)
    old = M.make_records(rng, pic, far=far, edge=edge, types=list(types))
    recs = np.zeros(len(old), REC)
    for name in M.REC.names:
        if name != "pad":
            recs[name] = old[name]
    recs["mcsel"] = rng.random(len(recs)) < mcsel
    pic.recs = recs[rng.random(len(recs)) >= intra]
    p = pic.p
    pic.sprite = params if params is not None else random_params(rng, p["width"], p["height"], mb_w, mb_h, p["h_edge_pos"], p["v_edge_pos"])
    return pic


def sprite_array(pic):
    acc, pts, off, d = pic.sprite
    return np.array([acc, pts] + [x for row in off for x in row] + [x for row in d for x in row], np.int32)


# ------------------------------------------------------------------------------------------------------------------------------- runners

def _bind(fn):
    fn.restype = C.c_int
    fn.argtypes = [C.c_void_p] * 5 + [C.c_void_p, C.c_size_t, C.c_void_p]
    return fn


def ref_lib():
    """the reference (ref_mpvmc_gmc_picture), or None where oracle/_ref was not built"""
    lib = loader.ref_lib("mpvgmc")
    if lib is None:
        return None
    lib.gmc_picture = _bind(lib.ref_mpvmc_gmc_picture)
    for name in ("ref_mpegvideodsp_init", "ref_mpegvideodsp_layout"):
        getattr(lib, name).argtypes = [C.c_void_p]
        getattr(lib, name).restype = None
    return lib


class _Port:
    def __init__(self):
        lib = loader.port().lib
        self.gmc_picture = _bind(lib.orc_mpvgmc_picture)
        self.gmc1, self.gmc = lib.orc_gmc1, lib.orc_gmc
        self.gmc1.argtypes = [C.c_void_p, C.c_void_p] + [C.c_int] * 5
        self.gmc.argtypes = [C.c_void_p, C.c_void_p] + [C.c_int] * 12


def port_lib():
    return _Port()


def checker_lib():
    return ref_lib() or port_lib()


def run_ref(lib, pic):
    """the reference or the port over an S-VOP's accepted records (a picture without .sprite: the plain path); returns its planes"""
    if getattr(pic, "sprite", None) is None:
        return M.run_ref(M.ref_lib() or M.port_lib(), pic)
    f = [a.copy() for a in pic.frame]
    recs, prm, sp = np.ascontiguousarray(pic.recs[pic.accepted()]), pic.prm(), sprite_array(pic)
    p = lambda planes: (C.c_void_p * 3)(*[a.ctypes.data for a in planes])
    assert lib.gmc_picture(p(f), p(f), p(pic.last), p(pic.next), prm.ctypes.data, recs.ctypes.data, len(recs), sp.ctypes.data) == 0
    return f


def set_sprite(s, pic):
    """the sprite fields of an FFMpvMCPicture from pic.sprite (a picture without one stays as it is)"""
    if getattr(pic, "sprite", None) is None:
        return s
    acc, pts, off, d = pic.sprite
    s.sprite, s.sprite_warping_accuracy, s.real_sprite_warping_points = 1, acc, pts
    for i in range(2):
        for k in range(2):
            s.sprite_offset[i][k], s.sprite_delta[i][k] = off[i][k], d[i][k]
    return s


def structs(pics, frames, recs):
    from libav_b200 import tables
    arr = (tables.FFMpvMCPicture * len(pics))()
    for i, pic in enumerate(pics):
        arr[i] = set_sprite(M.picture_struct(pic, frames[i], frames[i], [a.ctypes.data for a in pic.last], [a.ctypes.data for a in pic.next],
                                             recs[i].ctypes.data, len(recs[i])), pic)
    return arr


def run_sim(lib, pics):
    """the host-compiled product over the pictures in one call; returns (frames, rejected)"""
    frames = [[a.copy() for a in pic.frame] for pic in pics]
    recs = [np.ascontiguousarray(p.recs) for p in pics]
    arr = structs(pics, [[a.ctypes.data for a in f] for f in frames], recs)
    rej = np.zeros(1, np.uint32)
    rc = lib.ff_mpv_motion_batch_cuda(C.cast(arr, C.c_void_p), len(pics), rej.ctypes.data, None)
    assert rc == 0, lib.avb200_last_error()
    return frames, int(rej[0])


class GpuSvops(M.GpuPictures):
    """GpuPictures with the sprite fields of the pictures that have them"""

    def __init__(self, pics):
        super().__init__(pics)
        for i, p in enumerate(pics):
            set_sprite(self.arr[i], p)
