"""Pictures and records for the H.263 overlapped block motion compensation tests (tests/test_mpv_obmc_cpu.py, tests/test_gpu_mpv_obmc.py):
H.263 half-sample P pictures of tests/mpv_mc_cases.py with one FFMpvOBMCRecord per record, and the ways of running them -- the reference's
apply_obmc through the real ff_mpv_motion (oracle/_ref/libmpvobmcref.so), its plain-C restatement (oracle/port/orc_mpvobmc.c), the product
compiled for the host (tests/hostsim/h263_hostsim.cpp) and the product on the GPU."""
import ctypes as C
import os

import numpy as np

import mpv_mc_cases as M

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
OBMC_REF = os.path.join(ROOT, "oracle", "_ref", "libmpvobmcref.so")
OBMC = np.dtype([("mv", "<i2", (4, 2)), ("top", "<i2", (2, 2)), ("left", "<i2", (2, 2)), ("right", "<i2", (2, 2)),
                 ("mb_type_top", "<u4"), ("mb_type_left", "<u4"), ("mb_type_right", "<u4")])
assert OBMC.itemsize == 52
MB_TYPE_INTRA, MB_TYPE_L0_16X16 = 1, (1 << 3) | (1 << 12)


def obmc_picture(rng, mb_w, mb_h, no_rnd=0, b=0, ragged=0, intra=0.2, stale=0.3, far=0.1, edge=0.4):
    """an H.263 P (or B) picture with forward-only 16X16 / 8X8 records and their OBMC records.  Each record's own entries are its vectors
    (all four the one vector for 16X16); a neighbour's entries are that macroblock's vectors, or -- with probability `stale`, and always
    where the neighbour has no record -- other vectors (what the tables held from an earlier picture); neighbours are intra with
    probability `intra`.  ragged: 1 MPEG-4-style size not a multiple of 16, 2 H.263 custom size"""
    kw = dict(width=16 * mb_w - 5, height=16 * mb_h - 3, custom_edges=ragged == 2) if ragged else {}
    pic = M.Picture(rng, 2, mb_w, mb_h, no_rnd=no_rnd, b=b, **kw)
    M.make_records(rng, pic, far=far, edge=edge, types=[M.T16X16, M.T8X8])
    pic.recs["mv_dir"] = 1
    recs = pic.recs
    own = {}
    for r in recs:
        v = r["mv"][0].copy()
        if r["mv_type"] == M.T16X16:
            v[1:] = v[0]
        own[(int(r["mb_x"]), int(r["mb_y"]))] = v
    ob = np.zeros(len(recs), OBMC)

    def other(x, y):
        """two vectors of any kind for the macroblock at (x, y): small, far outside, or at / next to an edge"""
        v = np.zeros((2, 2), np.int16)
        for k in range(2):
            u = rng.random()
            kind = 1 if u < far else 2 if u < far + edge else 0
            v[k, 0] = M._component(rng, kind, 2, 16 * x, [pic.p["h_edge_pos"], pic.p["width"]], 8)
            v[k, 1] = M._component(rng, kind, 2, 16 * y, [pic.p["v_edge_pos"], pic.p["height"]], 8)
        return v

    for i, r in enumerate(recs):
        x, y = int(r["mb_x"]), int(r["mb_y"])
        o = ob[i]
        o["mv"] = own[(x, y)]
        for name, (nx, ny), rows in (("top", (x, y - 1), (2, 3)), ("left", (x - 1, y), (1, 3)), ("right", (x + 1, y), (0, 2))):
            src = own.get((nx, ny))
            o[name] = src[list(rows)] if src is not None and rng.random() >= stale else other(x, y)
            o["mb_type_" + name] = MB_TYPE_INTRA if rng.random() < intra else MB_TYPE_L0_16X16 | int(rng.integers(0, 1 << 20)) & ~7
    pic.obmc = ob
    return pic


def accepted(pic):
    return pic.accepted() & ((pic.recs["mv_dir"] & 3) == 1 if not pic.p["b_picture"] else True)


def _bind(fn):
    fn.restype = C.c_int
    fn.argtypes = [C.c_void_p] * 5 + [C.c_void_p, C.c_size_t, C.c_void_p]
    return fn


def ref_lib():
    if not os.path.exists(OBMC_REF):
        return None
    lib = C.CDLL(OBMC_REF)
    lib.picture = _bind(lib.ref_mpvmc_obmc_picture)
    return lib


class _Port:
    def __init__(self):
        from oracle import loader
        self.picture = _bind(loader.port().lib.orc_mpvobmc_picture)


def port_lib():
    return _Port()


def checker_lib():
    return ref_lib() or port_lib()


def run_ref(lib, pic):
    """the reference or the port over the picture's accepted records; returns the reconstructed planes"""
    f = [a.copy() for a in pic.frame]
    keep = accepted(pic)
    recs, ob, prm = np.ascontiguousarray(pic.recs[keep]), np.ascontiguousarray(pic.obmc[keep]), pic.prm()
    p = lambda planes: (C.c_void_p * 3)(*[a.ctypes.data for a in planes])
    assert lib.picture(p(f), p(f), p(pic.last), p(pic.next), prm.ctypes.data, recs.ctypes.data, len(recs), ob.ctypes.data) == 0
    return f


def structs(pics, frames, recs, obs, last=None, nxt=None):
    from libav_b200 import tables
    arr = (tables.FFMpvMCPicture * len(pics))()
    for i, pic in enumerate(pics):
        base = frames[i]
        s = M.picture_struct(pic, base, base, last[i], nxt[i], recs[i], len(pic.recs))
        s.obmc = 1
        s.obmc_recs = obs[i]
        arr[i] = s
    return arr


def run_sim(lib, pics):
    """the host-compiled product over the pictures in one call; returns (frames, rejected)"""
    frames = [[a.copy() for a in pic.frame] for pic in pics]
    recs = [np.ascontiguousarray(p.recs) for p in pics]
    obs = [np.ascontiguousarray(p.obmc) for p in pics]
    arr = structs(pics, [[a.ctypes.data for a in f] for f in frames], [r.ctypes.data for r in recs], [o.ctypes.data for o in obs],
                  [[a.ctypes.data for a in p.last] for p in pics], [[a.ctypes.data for a in p.next] for p in pics])
    rej = np.zeros(1, np.uint32)
    rc = lib.ff_mpv_motion_batch_cuda(C.cast(arr, C.c_void_p), len(pics), rej.ctypes.data, None)
    assert rc == 0, lib.hostsim_last_error()
    return frames, int(rej[0])
