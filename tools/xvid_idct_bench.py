#!/usr/bin/env python
"""xvid_idct_bench.py -- the Xvid IDCT's batched put against the simple IDCT's, alone and fused behind the h263_intra inverse quantiser,
on bench.py's idct_put buffers (2^20 dense int16 blocks into an 8192x8192 frame, TILES_PER_ROW 1024, bench.py's rotating buffer sets).

  python tools/xvid_idct_bench.py [--rounds 7] [--steps 200] [--warmup 20] [--arms simple,xvid,dq_simple,dq_xvid] [--out FILE.json]

  simple     ff_simple_idct_batch_cuda, mode 0 (put)
  xvid       ff_xvid_idct_batch_cuda, mode 0 (put)
  dq_simple  ff_mpeg_dequant_idct_batch_cuda, kind 5 (h263_intra)
  dq_xvid    ff_mpeg_dequant_xvid_idct_batch_cuda, kind 5 (h263_intra)

The arms run alternately (A B C D A B C D ...); each round times `steps` launches with CUDA events after `warmup` untimed ones.  Printed per
arm: the median and the best ms per step over the rounds, Gpixel/s, the algorithmic bytes (128 B of coefficients in + 64 B of pixels out per
block, + the 4-byte record for the fused arms) over the 3.35 TB/s of the H100 SXM data sheet, and the spread (max - min) / median.  The
card's name, power limit and maximum SM clock come from a read-only nvidia-smi query in the same run.  After the timed region every arm's
frame is compared with the CPU checker (the compiled reference when oracle/_ref travelled, else the port).  Without a GPU it fails.
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

ARMS = ("simple", "xvid", "dq_simple", "dq_xvid")
HBM_TBS = 3.35
KIND = 5                                     # h263_intra: what an MPEG-4 decoder's put_dct runs


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=30).stdout.strip()
    except Exception as e:          # the numbers still stand; say that the card could not be read
        out = "nvidia-smi unavailable: %s" % e
    return out.splitlines()[0] if out else "unknown"


def xvid_checker():
    """the Xvid batch of the compiled reference (oracle/_ref/libxvidref.so) if present, else of the port"""
    from oracle import loader
    path = os.path.join(ROOT, "oracle", "_ref", "libxvidref.so")
    if os.path.exists(path):
        f = C.CDLL(path).ref_xvid_idct_batch
        f.argtypes = [C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_ssize_t, C.c_size_t]
        return (lambda mode, b, fr, off, stride, n: f(mode, b, fr, off, stride, n)), "reference"
    f = loader.port().lib.orc_xvid_idct_batch
    f.argtypes = [C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_ssize_t, C.c_size_t, C.c_int]
    return (lambda mode, b, fr, off, stride, n: f(mode, b, fr, off, stride, n, os.cpu_count() or 1)), "port"


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
        raise SystemExit("xvid_idct_bench.py needs a GPU")
    torch.cuda.set_device(0)
    L.init(0)
    lib = L.lib
    stream = torch.cuda.current_stream().cuda_stream
    wl = bench.make_idct_workload(torch, L, stream, 0)
    d_blocks, d_frame = wl["keep"][0], wl["keep"][1]
    nbuf, n, tpr = len(d_blocks), bench.N_BLOCKS, bench.TILES_PER_ROW
    stride = tpr * 8

    # h263_intra records: qscale 1..31, last index 0..63, luma dc_scale, no AC prediction; the zigzag scan
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
        elif arm == "dq_simple":
            rc = lib.ff_mpeg_dequant_idct_batch_cuda(KIND, C.byref(t), d_rec.data_ptr(), b, f, None, stride, n, tpr, 0, stream)
        else:
            rc = lib.ff_mpeg_dequant_xvid_idct_batch_cuda(KIND, C.byref(t), d_rec.data_ptr(), b, f, None, stride, n, tpr, 0, stream)
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

    # after the timed region: every arm's frame (buffer 0) against the CPU checker, all 2^20 blocks
    blocks_h = d_blocks[0].cpu().numpy()
    i = np.arange(n, dtype=np.uint64)
    off = ((i // tpr) * 8 * stride + (i % tpr) * 8).astype(np.uint32)
    chk = loader.ref() or loader.port()
    xbatch, xkind = xvid_checker()
    deq = None
    if any(a.startswith("dq_") for a in names):
        deq = blocks_h.copy()
        intra = np.array(t.intra_matrix[:], np.uint16); inter = np.array(t.inter_matrix[:], np.uint16)
        for j in range(n):
            b = deq[j]
            chk.mpeg_dequant(KIND, b.ctypes.data_as(C.c_void_p), 0, int(rec["qscale"][j]), int(rec["last"][j]), 8, 8,
                             intra.ctypes.data_as(C.c_void_p), inter.ctypes.data_as(C.c_void_p), 0, 0, 0)
    verified = {}
    for a in names:
        d_frame[0].zero_()
        launch(a, 0)
        torch.cuda.synchronize()
        got = d_frame[0].cpu().numpy()
        want = np.zeros_like(got)
        src = np.ascontiguousarray((deq if a.startswith("dq_") else blocks_h).copy())
        if a.endswith("xvid"):
            xbatch(0, src.ctypes.data, want.ctypes.data, off.ctypes.data, stride, n)
        else:
            chk.idct_batch(0, src.ctypes.data_as(C.c_void_p), want.ctypes.data_as(C.c_void_p), off.ctypes.data_as(C.c_void_p), stride, n,
                           os.cpu_count() or 1)
        if not np.array_equal(got, want):
            raise SystemExit("xvid_idct_bench.py: arm %s differs from the CPU checker" % a)
        verified[a] = "all 2^20 blocks == %s" % (xkind if a.endswith("xvid") else chk.prefix.rstrip("_"))

    res = {"card": gpu, "rounds": args.rounds, "steps": args.steps, "blocks": n, "verified": verified, "arms": {}}
    print("card (name, power limit, max SM clock): %s" % gpu)
    print("%-10s %9s %9s %9s %8s %8s" % ("arm", "ms/step", "best", "Gpix/s", "%HBM", "spread"))
    for a in names:
        tt = sorted(times[a])
        med = tt[len(tt) // 2]
        spread = (tt[-1] - tt[0]) / med
        nbytes = n * (bench.IDCT_BYTES_PER_BLOCK + (4 if a.startswith("dq_") else 0))
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
