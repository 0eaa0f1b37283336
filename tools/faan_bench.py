#!/usr/bin/env python
"""faan_bench.py -- the FAAN transforms against the integer ones on bench.py's idct_put buffers (2^20 dense int16 blocks into an 8192x8192
frame, TILES_PER_ROW 1024, bench.py's rotating buffer sets).

  python tools/faan_bench.py [--rounds 7] [--steps 200] [--warmup 20] [--arms simple,xvid,faan,dq_faan,fdct_islow,fdct_faan] [--out FILE.json]

  simple      ff_simple_idct_batch_cuda, mode 0 (put)
  xvid        ff_xvid_idct_batch_cuda, mode 0 (put)
  faan        ff_faanidct_batch_cuda, mode 0 (put)
  dq_faan     ff_mpeg_dequant_faanidct_batch_cuda, kind 5 (h263_intra)
  fdct_islow  ff_fdct_batch_cuda 0 (ff_jpeg_fdct_islow_8), in place on a copy of the blocks
  fdct_faan   ff_fdct_batch_cuda 6 (ff_faandct), in place on the same copy

The arms run alternately; each round times `steps` launches with CUDA events after `warmup` untimed ones.  Printed per arm: the median and
the best ms per step over the rounds, Gpixel/s, the algorithmic bytes (put: 128 B of coefficients in + 64 B of pixels out per block, + the
4-byte record for the fused arm; in-place fdct: 256 B) over the 3.35 TB/s of the H100 SXM data sheet, and the spread (max - min) / median.
The card's name, power limit and maximum SM clock come from a read-only nvidia-smi query in the same run.  After the timed region every
arm's output is compared with the CPU checker (the compiled reference; the simple arm also accepts the port).  Without a GPU it fails.
"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

ARMS = ("simple", "xvid", "faan", "dq_faan", "fdct_islow", "fdct_faan")
HBM_TBS = 3.35
KIND = 5                                     # h263_intra: what an MPEG-4 decoder's put_dct runs

from xvid_idct_bench import card, xvid_checker      # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=7)
    ap.add_argument("--steps", type=int, default=200)
    ap.add_argument("--warmup", type=int, default=20)
    ap.add_argument("--arms", default=",".join(ARMS), help="comma-separated arm names")
    ap.add_argument("--out", help="also write the results as JSON to this file")
    args = ap.parse_args()
    names = args.arms.split(",")
    for n in names:
        if n not in ARMS:
            raise SystemExit("unknown arm %r (have: %s)" % (n, ", ".join(ARMS)))

    import torch
    import libav_b200._lib as L
    from libav_b200 import synth, tables
    from oracle import loader
    import bench
    if not torch.cuda.is_available():
        raise SystemExit("faan_bench.py needs a GPU")
    ref = loader.ref()
    if ref is None:
        raise SystemExit("faan_bench.py checks against oracle/_ref, which is not built here")
    torch.cuda.set_device(0)
    L.init(0)
    lib = L.lib
    stream = torch.cuda.current_stream().cuda_stream
    wl = bench.make_idct_workload(torch, L, stream, 0)
    d_blocks, d_frame = wl["keep"][0], wl["keep"][1]
    nbuf, n, tpr = len(d_blocks), bench.N_BLOCKS, bench.TILES_PER_ROW
    stride = tpr * 8
    d_fdct = d_blocks[0].clone()

    r = np.random.RandomState(5)
    rec = np.zeros(n, np.dtype([("qscale", "u1"), ("last", "i1"), ("dc", "u1"), ("flags", "u1")]))
    rec["qscale"] = r.randint(1, 32, n); rec["last"] = r.randint(0, 64, n); rec["dc"] = 8
    t = tables.FFMpegDequantTables()
    perm, rend = synth.zigzag_scan_tables()
    for k in range(64):
        t.intra_matrix[k] = t.inter_matrix[k] = 16
        t.permutated[k], t.raster_end[k] = int(perm[k]), int(rend[k])
    d_rec = torch.from_numpy(rec.view(np.uint8).reshape(-1)).cuda()

    def launch(arm, i):
        k = i % nbuf
        b, f = d_blocks[k].data_ptr(), d_frame[k].data_ptr()
        if arm == "simple":
            rc = lib.ff_simple_idct_batch_cuda(0, b, f, None, stride, n, tpr, 0, stream)
        elif arm == "xvid":
            rc = lib.ff_xvid_idct_batch_cuda(0, b, f, None, stride, n, tpr, 0, stream)
        elif arm == "faan":
            rc = lib.ff_faanidct_batch_cuda(0, b, f, None, stride, n, tpr, 0, stream)
        elif arm == "dq_faan":
            rc = lib.ff_mpeg_dequant_faanidct_batch_cuda(KIND, C.byref(t), d_rec.data_ptr(), b, f, None, stride, n, tpr, 0, stream)
        else:
            rc = lib.ff_fdct_batch_cuda(6 if arm == "fdct_faan" else 0, d_fdct.data_ptr(), n, stream)
        L.check(rc, arm)

    def timed(arm):
        for i in range(args.warmup):
            launch(arm, i)
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for i in range(args.steps):
            launch(arm, i)
        e1.record()
        torch.cuda.synchronize()
        L.check(0 if not L.last_error() else -1, "arm " + arm)
        return e0.elapsed_time(e1) / args.steps

    gpu = card()
    times = {a: [] for a in names}
    for _ in range(args.rounds):
        for a in names:
            times[a].append(timed(a))

    # after the timed region: every arm's output (buffer 0) against the CPU checker, all 2^20 blocks
    blocks_h = d_blocks[0].cpu().numpy().reshape(n, 64)
    i = np.arange(n, dtype=np.uint64)
    off = ((i // tpr) * 8 * stride + (i % tpr) * 8).astype(np.uint32)
    xbatch, _ = xvid_checker()
    rl = ref.lib
    for name, args_ in (("ff_faanidct_put", [C.c_void_p, C.c_ssize_t, C.c_void_p]), ("ff_faandct", [C.c_void_p]), ("ref_fdct", [C.c_int, C.c_void_p])):
        getattr(rl, name).restype, getattr(rl, name).argtypes = None, args_
    verified = {}
    for a in names:
        if a.startswith("fdct"):
            d_fdct.copy_(d_blocks[0])
            launch(a, 0)
            torch.cuda.synchronize()
            got = d_fdct.cpu().numpy().reshape(n, 64)
            want = np.ascontiguousarray(blocks_h.copy())
            for j in range(n):
                p = want.ctypes.data + 128 * j
                if a == "fdct_faan":
                    rl.ff_faandct(p)
                else:
                    rl.ref_fdct(0, p)
        else:
            d_frame[0].zero_()
            launch(a, 0)
            torch.cuda.synchronize()
            got = d_frame[0].cpu().numpy()
            want = np.zeros_like(got)
            src = np.ascontiguousarray(blocks_h.copy())
            if a == "dq_faan":
                intra = np.array(t.intra_matrix[:], np.uint16); inter = np.array(t.inter_matrix[:], np.uint16)
                for j in range(n):
                    ref.mpeg_dequant(KIND, C.c_void_p(src.ctypes.data + 128 * j), 0, int(rec["qscale"][j]), int(rec["last"][j]), 8, 8,
                                     intra.ctypes.data_as(C.c_void_p), inter.ctypes.data_as(C.c_void_p), 0, 0, 0)
            if a in ("faan", "dq_faan"):
                for j in range(n):
                    rl.ff_faanidct_put(want.ctypes.data + int(off[j]), stride, src.ctypes.data + 128 * j)
            elif a == "xvid":
                xbatch(0, src.ctypes.data, want.ctypes.data, off.ctypes.data, stride, n)
            else:
                ref.idct_batch(0, src.ctypes.data_as(C.c_void_p), want.ctypes.data_as(C.c_void_p), off.ctypes.data_as(C.c_void_p), stride, n,
                               os.cpu_count() or 1)
        if not np.array_equal(got, want):
            raise SystemExit("faan_bench.py: arm %s differs from the reference" % a)
        verified[a] = "all 2^20 blocks == reference"

    res = {"card": gpu, "rounds": args.rounds, "steps": args.steps, "blocks": n, "verified": verified, "arms": {}}
    print("card (name, power limit, max SM clock): %s" % gpu)
    print("%-10s %9s %9s %9s %8s %8s" % ("arm", "ms/step", "best", "Gpix/s", "%HBM", "spread"))
    for a in names:
        tt = sorted(times[a])
        med = tt[len(tt) // 2]
        spread = (tt[-1] - tt[0]) / med
        nbytes = n * (256 if a.startswith("fdct") else bench.IDCT_BYTES_PER_BLOCK + (4 if a.startswith("dq_") else 0))
        gpix = n * 64 / (med * 1e-3) / 1e9
        frac = nbytes / (med * 1e-3) / (HBM_TBS * 1e12)
        print("%-10s %9.4f %9.4f %9.1f %7.1f%% %7.2f%%" % (a, med, tt[0], gpix, 100 * frac, 100 * spread))
        res["arms"][a] = {"ms_per_step": med, "best_ms": tt[0], "gpix_per_s": gpix, "hbm_fraction": frac, "alg_bytes": nbytes, "spread": spread,
                          "times": times[a]}
    print("verified: %s" % verified)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(res, f, indent=1)
    return 0


if __name__ == "__main__":
    sys.exit(main())
