"""Build recipe for the native pieces (called by __graft_entry__.build() and usable as a script).

  libav_b200/libavdsp_b200.so   the product: hand-written sm_90a kernels + the C-ABI (nvcc)
  oracle/liboracle_port.so      TEST ONLY: plain-C restatement of the reference path (gcc)
  oracle/_ref/libavref.so       TEST ONLY: the unmodified reference compiled from /root/reference,
                                only when that tree is present (never on the GPU box)
  oracle/_ref/libxvidref.so     TEST ONLY: the reference's Xvid IDCT, same conditions
  oracle/_ref/libmpvmcref.so    TEST ONLY: the reference's mpegvideo motion compensation, same conditions
  oracle/_ref/libmpvqref.so     TEST ONLY: the reference's encoder quantisers (plain, trellis, noise reduction), same conditions
  oracle/_ref/libmpvobmcref.so  TEST ONLY: the reference's H.263 overlapped block motion compensation (apply_obmc), same conditions
  oracle/_ref/libh263ref.so     TEST ONLY: the reference's H.263 deblocking filter (H263DSPContext, ff_h263_loop_filter), same conditions
All outputs are in-tree so they travel to the GPU box with the snapshot.
"""
import glob
import os
import shutil
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "libav_b200", "csrc")
LIB = os.path.join(ROOT, "libav_b200", "libavdsp_b200.so")
ORACLE_PORT = os.path.join(ROOT, "oracle", "liboracle_port.so")
ORACLE_REF = os.path.join(ROOT, "oracle", "_ref", "libavref.so")
REFERENCE = "/root/reference"

GENCODE = ["-gencode", "arch=compute_90a,code=sm_90a"]      # H100 (Hopper)
NVCC_FLAGS = GENCODE + ["-lineinfo", "-O3", "-std=c++17",
              "-Xcompiler", "-fPIC", "-cudart", "static"]


def _newer(target, sources):
    if not os.path.exists(target):
        return True
    t = os.path.getmtime(target)
    return any(os.path.getmtime(s) > t for s in sources)


def _run(cmd, **kw):
    r = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, **kw)
    if r.returncode != 0:
        sys.stderr.write(r.stdout)
        raise RuntimeError("command failed: " + " ".join(cmd))
    return r.stdout


def build_cuda(force=False, verbose=False):
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    srcs = sorted(glob.glob(os.path.join(CSRC, "*.cu")))
    deps = srcs + glob.glob(os.path.join(CSRC, "*.h")) + glob.glob(os.path.join(CSRC, "*.cuh")) + \
        glob.glob(os.path.join(ROOT, "include", "*.h"))
    if not force and not _newer(LIB, deps):
        return LIB
    objdir = os.path.join(CSRC, "build")
    os.makedirs(objdir, exist_ok=True)
    procs = []
    objs = []
    for s in srcs:
        o = os.path.join(objdir, os.path.basename(s)[:-3] + ".o")
        objs.append(o)
        if force or _newer(o, [s] + [d for d in deps if not d.endswith(".cu")]):
            cmd = [nvcc] + NVCC_FLAGS + (["-Xptxas", "-v"] if verbose else []) + ["-c", s, "-o", o]
            procs.append((cmd, subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)))
    for cmd, p in procs:
        out, _ = p.communicate()
        if verbose or p.returncode:
            sys.stderr.write(out)
        if p.returncode:
            raise RuntimeError("nvcc failed: " + " ".join(cmd))
    _run([nvcc] + GENCODE + ["-shared", "-cudart", "static", "-o", LIB] + objs)
    return LIB


def build_oracle_port(force=False):
    srcs = sorted(glob.glob(os.path.join(ROOT, "oracle", "port", "*.c")))
    deps = srcs + [os.path.join(ROOT, "oracle", "oracle_api.h")]
    if not force and not _newer(ORACLE_PORT, deps):
        return ORACLE_PORT
    _run(["gcc", "-O2", "-fPIC", "-shared", "-std=gnu99", "-Wall", "-Wno-comment", "-fwrapv", "-o", ORACLE_PORT] + srcs + ["-lm", "-lpthread"])
    return ORACLE_PORT


def build_oracle_ref(force=False):
    """Compile the reference's own C sources (read in place) with oracle/refbuild/Makefile: libavref.so, its timing-only SIMD
    flavour and the satellite libraries of single features, all in one make run."""
    if not os.path.isdir(REFERENCE):
        return ORACLE_REF if os.path.exists(ORACLE_REF) else None
    if force:
        shutil.rmtree(os.path.join(ROOT, "oracle", "_ref"), ignore_errors=True)
    _run(["make", "-s", "-j8", "-C", os.path.join(ROOT, "oracle", "refbuild"), "REF=" + REFERENCE])
    return ORACLE_REF


def build_all(force=False, verbose=False):
    return {"cuda": build_cuda(force, verbose), "oracle_port": build_oracle_port(force), "oracle_ref": build_oracle_ref(force)}


if __name__ == "__main__":
    print(build_all(force="--force" in sys.argv, verbose="-v" in sys.argv))
