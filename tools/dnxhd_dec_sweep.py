#!/usr/bin/env python
"""dnxhd_dec_sweep.py -- the entropy stage's launch shape of ff_dnxhd_decode_frames_cuda: active lanes per warp, at 16 and 64 1920x1080
packets per call (CIDs 1238, 8 bit, and 1235, 10 bit).

  python tools/dnxhd_dec_sweep.py [--steps 10] [--out FILE.json]

Each shape is a copy of libav_b200/csrc/dnxhd_dec.cu whose dd_lanes() returns that count, compiled with runtime.cu into a small library in
a temporary directory (nothing is written in the tree); the library as built is timed too.  Each call is timed alone with CUDA events after
a warm-up call, median over steps; every shape's frames are compared with the built library's.  The card's name, power limit and maximum
SM clock are read in the same run.  Without a GPU it fails.
"""
import argparse
import ctypes as C
import json
import os
import re
import shutil
import subprocess
import sys
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
sys.path.insert(0, os.path.join(ROOT, "tests"))

from xvid_idct_bench import card      # noqa: E402

LANES = (1, 2, 3, 4, 6, 8, 16, 32)


def build_variants(tmp):
    """{lanes: path of a library whose entropy launch has that many active lanes per warp}"""
    from libav_b200 import build
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    csrc = os.path.join(ROOT, "libav_b200", "csrc")
    src = open(os.path.join(csrc, "dnxhd_dec.cu")).read()
    body = re.compile(r"(int dd_lanes\(int rows\)\n\{\n).*?(\n\}\n)", re.S)
    assert body.search(src)
    rt = os.path.join(tmp, "runtime.o")
    subprocess.run([nvcc] + build.NVCC_FLAGS + ["-c", os.path.join(csrc, "runtime.cu"), "-o", rt], check=True)
    procs, out = [], {}
    for lanes in LANES:
        name = "dd_%d" % lanes
        tmp_cu = os.path.join(tmp, name + ".cu")
        open(tmp_cu, "w").write(body.sub(lambda m: m.group(1) + "    (void)rows;\n    return %d;" % lanes + m.group(2), src))
        obj, lib = os.path.join(tmp, name + ".o"), os.path.join(tmp, name + ".so")
        cmd = [nvcc] + build.NVCC_FLAGS + ["-I", csrc, "-c", tmp_cu, "-o", obj]
        procs.append((subprocess.Popen(cmd), obj, lib, lanes))
    for p, obj, lib, key in procs:
        assert p.wait() == 0, key
        subprocess.run([nvcc] + build.GENCODE + ["-shared", "-cudart", "static", "-o", lib, obj, rt], check=True)
        out[key] = lib
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import torch
    assert torch.cuda.is_available(), "needs a GPU"
    import __graft_entry__ as g
    g.build()
    import libav_b200._lib as L
    L.init(0)
    import dnxhd_dec_util as D
    import dnxhd_enc_util as E
    from libav_b200 import tables
    dref, eref = D.ref(), E.ref()
    cids, ncids, _ = D.cid_table(dref)
    gpu = card()
    print("card (name, power limit, max SM clock): %s" % gpu)
    tmp = tempfile.mkdtemp()
    try:
        libs = {"built": L.lib}
        for key, path in build_variants(tmp).items():
            lib = C.CDLL(path)
            for name, (restype, argtypes) in L.PROTOTYPES.items():
                if name.startswith("ff_dnxhd_") and hasattr(lib, name):
                    getattr(lib, name).restype, getattr(lib, name).argtypes = restype, argtypes
            libs["lanes %d" % key] = lib
        dev = torch.device("cuda")
        results = {"card": gpu, "ms_per_call": {}}
        for cid in (1238, 1235):
            pk = D.real_packets(eref, cid, ["natural", "noise"], seed=5)
            ret, info = D.info_of(L.lib, pk[0], cids, ncids)
            assert ret == 0
            bpp = 1 if info.pix_fmt == 4 else 2
            lss = [info.width * bpp, info.width // 2 * bpp, info.width // 2 * bpp]
            for n in (16, 64):
                host = [np.frombuffer(pk[k % 2], np.uint8).copy() for k in range(n)]
                dpk = [torch.from_numpy(h).to(dev) for h in host]
                want = None
                for name, lib in libs.items():
                    planes = [[torch.full((info.lines, ls), D.SENTINEL, dtype=torch.uint8, device=dev) for ls in lss] for _ in range(n)]
                    works = []
                    for k in range(n):
                        w = tables.FFDnxhdDecodeWork()
                        w.pkt_host, w.pkt, w.size = host[k].ctypes.data, dpk[k].data_ptr(), len(host[k])
                        for p in range(3):
                            w.data[p], w.linesize[p], w.lines[p] = planes[k][p].data_ptr(), lss[p], info.lines
                        works.append(w)
                    arr = (tables.FFDnxhdDecodeWork * n)(*works)
                    need = lib.ff_dnxhd_decode_workspace_cuda(arr, n, cids, ncids)
                    ws = torch.empty(need, dtype=torch.uint8, device=dev)
                    st = C.c_void_p(torch.cuda.current_stream().cuda_stream)

                    def call():
                        assert lib.ff_dnxhd_decode_frames_cuda(arr, n, cids, ncids, C.c_void_p(ws.data_ptr()), need, st) == 0
                    call(); torch.cuda.synchronize()
                    ts = []
                    for _ in range(a.steps):
                        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                        e0.record(); call(); e1.record(); e1.synchronize()
                        ts.append(e0.elapsed_time(e1))
                    got = [torch.cat([x.flatten() for x in f]).cpu().numpy() for f in planes]
                    if want is None:
                        want = got
                    assert all(np.array_equal(x, y) for x, y in zip(got, want)), (name, cid, n)
                    ms = float(np.median(ts))
                    results["ms_per_call"]["%d n=%d %s" % (cid, n, name)] = ms
                    print("%d n=%2d %-20s %8.3f ms/call  %6.0f frames/s  spread %.2f" % (cid, n, name, ms, n / ms * 1e3,
                                                                                         (max(ts) - min(ts)) / ms))
        if a.out:
            os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
            json.dump(results, open(a.out, "w"), indent=1)
    finally:
        shutil.rmtree(tmp, ignore_errors=True)


if __name__ == "__main__":
    main()
