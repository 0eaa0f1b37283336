"""TEST INFRASTRUCTURE.  Builds and loads tests/hostsim/libhostsim.so: every unit tests/hostsim/*_hostsim.cpp (the product's
thread-independent kernels and their host code, compiled unchanged as host C++ against tests/hostsim/shim/, and their one runtime,
runtime_hostsim.cpp) in one library.  load() rebuilds it when any product source, public header or file under tests/hostsim/ is newer, compiling the units in
parallel.  Every file is written under a name of its own process and renamed into place, so test processes that build at the same time
never see a half-written file.  Only the CPU suite loads this library; the product never does."""
import ctypes as C
import glob
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
HS = os.path.join(HERE, "hostsim")
GEN = os.path.join(HS, "_gen")
CSRC = os.path.join(ROOT, "libav_b200", "csrc")
LIB = os.path.join(HS, "libhostsim.so")
CXXFLAGS = ["-O2", "-std=c++17", "-fPIC", "-x", "c++", "-DAVB_HOSTSIM", "-I", os.path.join(HS, "shim"), "-I", CSRC, "-Wno-unknown-pragmas"]

vp, sz, i32 = C.c_void_p, C.c_size_t, C.c_int
# the library's own entry points; the product's ABI symbols take their prototypes from libav_b200._lib.PROTOTYPES
HELPERS = {
    "hostsim_h264_mc": (i32, [vp, sz, vp, vp, vp, vp, i32, i32, i32, i32, i32]),
    "hostsim_h264_residual": (i32, [vp, sz, vp, sz, vp, vp, vp, vp, i32, i32]),
    "hostsim_h264_pred_init_hbd": (None, [vp, i32]),
    "hostsim_h264_pred_install_422": (None, [vp, i32]),
    "hostsim_idctdsp_init10": (None, [vp]),
    "hostsim_rgb_constants": (i32, [vp, vp, i32, i32, i32, i32]),
    "hostsim_h263_slot": (i32, [i32, vp, i32, i32]),
}

_lib = None


def _deps():
    srcs = [p for p in glob.glob(os.path.join(HS, "**"), recursive=True)
            if os.path.isfile(p) and not p.startswith(GEN + os.sep) and not p.endswith(".so") and ".tmp" not in p]
    return srcs + [os.path.abspath(__file__)] + glob.glob(os.path.join(ROOT, "include", "*.h")) + \
        [p for ext in ("cu", "cuh", "h") for p in glob.glob(os.path.join(CSRC, "*." + ext))]


def _stale():
    if not os.path.exists(LIB):
        return True
    t = os.path.getmtime(LIB)
    return any(os.path.getmtime(p) > t for p in _deps())


def _build():
    os.makedirs(GEN, exist_ok=True)
    tag = ".%d.tmp" % os.getpid()
    gen = os.path.join(GEN, "swscale_gen.cu")
    subprocess.run([sys.executable, os.path.join(HS, "gen_launches.py"), os.path.join(CSRC, "swscale.cu"), gen + tag], check=True)
    os.replace(gen + tag, gen)
    units = sorted(glob.glob(os.path.join(HS, "*_hostsim.cpp")))
    objs = [os.path.join(GEN, os.path.basename(u)[:-4] + tag + ".o") for u in units]
    try:
        procs = [subprocess.Popen(["g++"] + CXXFLAGS + ["-c", u, "-o", o]) for u, o in zip(units, objs)]
        failed = [u for u, p in zip(units, procs) if p.wait()]
        assert not failed, "host build failed: %s" % failed
        subprocess.run(["g++", "-shared", "-Wl,--no-undefined", "-o", LIB + tag] + objs, check=True)
        os.replace(LIB + tag, LIB)
    finally:
        for p in objs + [LIB + tag]:
            if os.path.exists(p):
                os.remove(p)


def load():
    """the library, built if it is missing or older than its sources, with prototypes set; one handle per process"""
    global _lib
    if _lib is None:
        if _stale():
            _build()
        from libav_b200 import _lib as product
        lib = C.CDLL(LIB)
        for name, (restype, argtypes) in list(product.PROTOTYPES.items()) + list(HELPERS.items()):
            if hasattr(lib, name):
                f = getattr(lib, name)
                f.restype, f.argtypes = restype, argtypes
        _lib = lib
    return _lib


def fresh():
    """load() with the error channel cleared, so that what a test reads from it is what its own calls left there"""
    lib = load()
    lib.avb200_clear_error()
    return lib
