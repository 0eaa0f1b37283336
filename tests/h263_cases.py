"""Pictures for the H.263 deblocking filter tests (tests/test_h263_cpu.py, tests/test_gpu_h263.py), and the ways of running them: the
reference's serial driver (ff_h263_loop_filter per macroblock in raster order, oracle/_ref/libh263ref.so), its two-pass plain-C
restatement (oracle/port/orc_h263.c), the product compiled for the host (tests/hostsim/h263_hostsim.cpp) and the product on the GPU.
Every plane buffer holds random bytes, its padding included: two rows above and below the macroblock-aligned plane and columns to the
right of it, so a kernel that writes outside the plane gives a different buffer."""
import ctypes as C
import os
import subprocess

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
H263_REF = os.path.join(ROOT, "oracle", "_ref", "libh263ref.so")
SIM_LIB = os.path.join(HERE, "hostsim", "libh263_hostsim.so")
MB_TYPE_SKIP = 1 << 11
PAD_ROWS = 2
DEFAULT_CHROMA_QSCALE = np.arange(32, dtype=np.uint8)              # ff_default_chroma_qscale_table (mpegvideodata.c): the identity
ANNEX_T_CHROMA_QSCALE = np.fromfile(os.path.join(HERE, "golden", "h263_annex_t_chroma_qscale.bin"), np.uint8)   # H.263 Table T.1
assert ANNEX_T_CHROMA_QSCALE.shape == (32,)


class LfPicture:
    """One reconstructed picture as the decoder leaves it before the loop filter: planes, mb_type (random bits besides MB_TYPE_SKIP, which
    the filter must ignore) and qscale_table, indexed mb_x + mb_y * mb_stride.  `bufs` are the whole plane buffers, padding included;
    `data` offsets address row 0 of each plane inside them."""

    def __init__(self, rng, mb_w, mb_h, skip=0.3, qmin=1, qmax=31, chroma=None, extra_cols=None, mb_stride=None):
        self.mb_w, self.mb_h = mb_w, mb_h
        self.mb_stride = mb_stride or mb_w + 1
        ex = int(rng.integers(0, 40)) if extra_cols is None else extra_cols
        self.ls, self.uvls = 16 * mb_w + ex, 8 * mb_w + ex // 2
        self.bufs = [rng.integers(0, 256, (16 * mb_h + 2 * PAD_ROWS, self.ls), dtype=np.uint8),
                     rng.integers(0, 256, (8 * mb_h + 2 * PAD_ROWS, self.uvls), dtype=np.uint8),
                     rng.integers(0, 256, (8 * mb_h + 2 * PAD_ROWS, self.uvls), dtype=np.uint8)]
        n = self.mb_stride * mb_h
        self.mb_type = rng.integers(0, 1 << 20, n, dtype=np.uint32) & ~np.uint32(MB_TYPE_SKIP)
        self.mb_type[rng.random(n) < skip] |= MB_TYPE_SKIP
        self.qscale = rng.integers(qmin, qmax + 1, n).astype(np.int8)
        self.chroma = DEFAULT_CHROMA_QSCALE if chroma is None else chroma

    @property
    def offs(self):
        return [PAD_ROWS * self.ls, PAD_ROWS * self.uvls, PAD_ROWS * self.uvls]

    def prm(self):
        return np.array([self.ls, self.uvls, self.mb_w, self.mb_h, self.mb_stride], np.int32)

    def struct(self, base):
        """FFH263LoopFilterPicture for buffers at `base` (host or device addresses of bufs), tables at the given addresses"""
        from libav_b200 import tables
        s = tables.FFH263LoopFilterPicture()
        for i in range(3):
            s.data[i] = base[i] + self.offs[i]
        s.linesize, s.uvlinesize, s.mb_width, s.mb_height, s.mb_stride = self.ls, self.uvls, self.mb_w, self.mb_h, self.mb_stride
        s.chroma_qscale_table[:] = [int(x) for x in self.chroma]
        return s


def _ptrs(bufs, offs):
    return (C.c_void_p * 3)(*[a.ctypes.data + o for a, o in zip(bufs, offs)])


def _bind(fn):
    fn.restype = C.c_int
    fn.argtypes = [C.c_void_p] * 5
    return fn


def ref_lib():
    """the reference's serial driver (ref_h263_loop_filter_picture), or None where oracle/_ref was not built"""
    if not os.path.exists(H263_REF):
        return None
    lib = C.CDLL(H263_REF)
    lib.picture = _bind(lib.ref_h263_loop_filter_picture)
    return lib


class _Port:
    def __init__(self):
        from oracle import loader
        lib = loader.port().lib
        self.picture = _bind(lib.orc_h263_loop_filter_picture)
        self.h_loop_filter, self.v_loop_filter = lib.orc_h263_h_loop_filter, lib.orc_h263_v_loop_filter
        for f in (self.h_loop_filter, self.v_loop_filter):
            f.restype, f.argtypes = None, [C.c_void_p, C.c_int, C.c_int]


def port_lib():
    return _Port()


def checker_lib():
    """the strongest checker available: the reference's serial driver where it was built, else the two-pass port (pinned to it)"""
    return ref_lib() or port_lib()


def run_serial(lib, pic):
    """the reference or the port over one picture; returns the filtered buffers (copies)"""
    b = [a.copy() for a in pic.bufs]
    mt, qs, ct, prm = pic.mb_type.copy(), pic.qscale.copy(), np.ascontiguousarray(pic.chroma, np.uint8), pic.prm()
    assert lib.picture(_ptrs(b, pic.offs), prm.ctypes.data, mt.ctypes.data, qs.ctypes.data, ct.ctypes.data) == 0
    return b


def sim_lib():
    """tests/hostsim/h263_hostsim.cpp built into its own library (under a temporary name, then renamed into place)"""
    hs = os.path.join(HERE, "hostsim")
    csrc = os.path.join(ROOT, "libav_b200", "csrc")
    src = os.path.join(hs, "h263_hostsim.cpp")
    deps = [src, os.path.join(hs, "mpv_mc_hostsim.cpp"), os.path.join(hs, "shim", "cuda_runtime.h"), os.path.join(csrc, "mpv_mc.cu"),
            os.path.join(csrc, "mpv_mc_block.cuh"), os.path.join(csrc, "h263_lf.cuh"), os.path.join(csrc, "common.cuh"),
            os.path.join(ROOT, "include", "avdsp_b200.h")]
    if not os.path.exists(SIM_LIB) or any(os.path.getmtime(d) > os.path.getmtime(SIM_LIB) for d in deps):
        tmp = "%s.%d.tmp" % (SIM_LIB, os.getpid())
        subprocess.run(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-x", "c++", "-DAVB_HOSTSIM", "-I", os.path.join(hs, "shim"), "-I", csrc,
                        "-Wno-unknown-pragmas", "-Wl,--no-undefined", "-o", tmp, src], check=True)
        os.replace(tmp, SIM_LIB)
    lib = C.CDLL(SIM_LIB)
    lib.ff_h263_loop_filter_batch_cuda.restype = C.c_int
    lib.ff_h263_loop_filter_batch_cuda.argtypes = [C.c_void_p, C.c_int, C.c_void_p]
    lib.ff_mpv_flush_pictures_cuda.restype = C.c_int
    lib.ff_mpv_flush_pictures_cuda.argtypes = [C.c_void_p, C.c_void_p]
    lib.hostsim_h263_slot.restype = C.c_int
    lib.hostsim_h263_slot.argtypes = [C.c_int, C.c_void_p, C.c_int, C.c_int]
    lib.hostsim_last_error.restype = C.c_char_p
    return lib


def host_structs(pics, bufs):
    """an FFH263LoopFilterPicture array over host buffers `bufs` (one list of three planes per picture)"""
    from libav_b200 import tables
    arr = (tables.FFH263LoopFilterPicture * len(pics))()
    for i, (pic, b) in enumerate(zip(pics, bufs)):
        s = pic.struct([a.ctypes.data for a in b])
        s.mb_type, s.qscale_table = pic.mb_type.ctypes.data, pic.qscale.ctypes.data
        arr[i] = s
    return arr


def run_sim(lib, pics):
    """the host-compiled product over all the pictures in one call; returns the filtered buffers"""
    bufs = [[a.copy() for a in pic.bufs] for pic in pics]
    arr = host_structs(pics, bufs)
    rc = lib.ff_h263_loop_filter_batch_cuda(C.cast(arr, C.c_void_p), len(pics), None)
    assert rc == 0, lib.hostsim_last_error()
    return bufs


class GpuLf:
    """the pictures' planes and tables in device memory, and the FFH263LoopFilterPicture array that describes them"""

    def __init__(self, pics):
        from libav_b200 import device, tables
        dev = lambda a: device.DevBuf.from_numpy(np.ascontiguousarray(a))
        self.pics, self.frames, self.keep = pics, [], []
        self.arr = (tables.FFH263LoopFilterPicture * len(pics))()
        for i, pic in enumerate(pics):
            fr = [dev(a) for a in pic.bufs]
            mt, qs = dev(pic.mb_type), dev(pic.qscale)
            self.frames.append(fr)
            self.keep += [mt, qs]
            s = pic.struct([b.ptr for b in fr])
            s.mb_type, s.qscale_table = mt.ptr, qs.ptr
            self.arr[i] = s

    def download(self):
        return [[b.download(np.uint8, a.shape) for b, a in zip(fr, pic.bufs)] for fr, pic in zip(self.frames, self.pics)]


def first_diff(got, want):
    for pl in range(3):
        if not np.array_equal(got[pl], want[pl]):
            yx = np.argwhere(got[pl] != want[pl])[0]
            return "plane %d first difference at buffer row %d col %d: %d vs %d" % (pl, yx[0], yx[1], got[pl][tuple(yx)], want[pl][tuple(yx)])
    return None


# ---------------------------------------------------------------------------------------------------------------------------- the slots

def slot_case(rng, vert, stride_sign, qscale, dkind):
    """a 12 x 12 buffer and the address of src inside it (row 4, column 4) for one slot call: the stride is 12 or -12, and the four
    samples of every line are built to put d = (p0 - p3 + 4 (p2 - p1)) / 8 in the chosen range of the filter (0: |d| < s, 1: s <= |d| < 2s,
    2: |d| >= 2s, 3: random, with clipping at 0 / 255 likely)"""
    buf = rng.integers(0, 256, (12, 12), dtype=np.uint8)
    s = [0, 1, 1, 2, 2, 3, 3, 4, 4, 4, 5, 5, 6, 6, 7, 7, 7, 8, 8, 8, 9, 9, 9, 10, 10, 10, 11, 11, 11, 12, 12, 12][qscale]
    for line in range(8):
        if dkind == 3:
            p = rng.integers(0, 256, 4)
            if rng.random() < 0.5:
                p = np.array(rng.choice([0, 1, 2, 253, 254, 255], 4))
        else:
            lo, hi = [(0, max(s, 1)), (s, 2 * s + 1), (2 * s, 80)][dkind]
            d = int(rng.integers(lo, max(hi, lo + 1))) * int(rng.choice([-1, 1]))
            p1 = int(rng.integers(40, 216))
            p0 = int(rng.integers(0, 256))
            p2 = int(np.clip(p1 + (2 * d + int(rng.integers(-1, 2))), 0, 255))
            p3 = int(np.clip(p0 + 4 * (p2 - p1) - 8 * d + int(rng.integers(-3, 4)), 0, 255))
            p = np.array([p0, p1, p2, p3])
        for i in range(4):
            if vert:
                buf[4 + line, 2 + i] = p[i]
            else:
                buf[2 + i, 4 + line] = p[i]
    if stride_sign < 0:
        buf = buf[::-1].copy()          # the same lines read upwards: src on row 7, stride -12
        return buf, 7 * 12 + 4, -12
    return buf, 4 * 12 + 4, 12
