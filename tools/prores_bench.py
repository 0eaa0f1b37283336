#!/usr/bin/env python
"""prores_bench.py -- ProRes reconstruction of sixteen 4096x2160 4:2:2 frames per call, coefficients from the reference encoder at the HQ
profile (two seeded source frames, each used for eight of the sixteen).

  python tools/prores_bench.py [--rounds 7] [--steps 10] [--frames 16] [--out FILE.json]

  picture      ff_prores_decode_pictures_cuda over the sixteen pictures (the decoder's flush point; one launch)
  picture_2x8  the same sixteen pictures as two calls of eight, back to back (two launches)
  picture8     ff_prores_decode_pictures_cuda over the first eight pictures
  batch8       ff_prores_idct_put_batch_cuda over the same eight pictures' blocks
  batch        ff_prores_idct_put_batch_cuda over the sixteen pictures' blocks, one matrix per block record, the same destinations
  idct10       ff_simple_idct10_batch_cuda mode 0 (put) over the same block count and destinations: the same transform without ProRes

The arms alternate within each round; every step restores the coefficients from a pristine copy outside the timed interval (batch and
idct10 write into them) and is timed alone with CUDA events.  Printed per arm: median and best ms per call, Gblocks/s, the algorithmic bytes
(picture: 128 B of coefficients in + 128 B of samples out = 256 B per block; batch and idct10: + 128 B written back = 384 B) over the
3.35 TB/s of the H100 SXM data sheet, and the spread (max - min) / median over rounds x steps.  The CPU baseline is prores_idct_put_c over
the same blocks on every host core (oracle/_ref/libproresref.so).  After the timed region the picture and batch arms' y / u / v planes are
compared with the reference decoder's.  A separate torch.profiler pass (CUDA activities, one call per arm, after the timed region)
lists each arm's kernels with their device durations and, for picture_2x8, the gap between the two launches.  The card's name, power
limit and maximum SM clock come from a read-only nvidia-smi query in the same run.  Without a GPU it fails.
"""
import argparse
import ctypes as C
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
sys.path.insert(0, os.path.join(ROOT, "tests"))

HBM_TBS = 3.35
W, H = 4096, 2160
ARMS = ("picture", "picture_2x8", "picture8", "batch8", "batch", "idct10")

from xvid_idct_bench import card      # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=7)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--frames", type=int, default=16)
    ap.add_argument("--out", help="also write the results as JSON to this file")
    args = ap.parse_args()

    import torch
    import libav_b200._lib as L
    from libav_b200 import tables
    import prores_util as U
    if not torch.cuda.is_available():
        raise SystemExit("prores_bench.py needs a GPU")
    ref = U.ref()
    if ref is None:
        raise SystemExit("prores_bench.py encodes and checks with oracle/_ref, which is not built here")
    ref.ref_prores_idct_put_batch.restype = C.c_int
    ref.ref_prores_idct_put_batch.argtypes = [C.c_void_p] * 5 + [C.c_ssize_t, C.c_size_t, C.c_int]
    torch.cuda.set_device(0)
    L.init(0)
    lib = L.lib
    stream = torch.cuda.current_stream().cuda_stream

    # two reference-encoded HQ frames, decoded by the reference with the work recorded; one frame layout with a common linesize so that
    # the batch arms address every plane with one pitch
    t0 = time.time()
    src = []
    for seed in (1, 2):
        fr = U.Frame(U.FMT_422, W, H, 0, seed)
        fr.ls = [fr.ls[0]] * 4
        o = 0
        fr.off = []
        for p in range(4):
            fr.off.append(o); o += fr.ls[p] * fr.H + 64
        fr.buf = np.zeros(o, np.uint8)
        pkt = U.encode(ref, U.FMT_422, W, H, 0, 3, seed)
        want, rec = U.decode(ref, fr, pkt)
        src.append((fr, want, rec, len(pkt)))
    print("encoded and decoded 2 frames with the reference in %.1f s (%d / %d bytes)" % (time.time() - t0, src[0][3], src[1][3]))
    fr = src[0][0]
    F, fbytes = args.frames, len(fr.buf)
    nb = src[0][2].n_blocks
    assert src[1][2].n_blocks == nb
    n = F * nb

    blocks = np.concatenate([src[k % 2][2].np_blocks for k in range(F)])
    qall = np.concatenate([src[k % 2][2].np_qmat for k in range(F)])
    qmats, qidx = np.unique(qall, axis=0, return_inverse=True)
    qidx = qidx.reshape(-1).astype(np.uint32)
    dst_off = np.concatenate([src[k % 2][2].np_dst + k * fbytes for k in range(F)]).astype(np.uint32)
    slices = [U.slice_table(src[k % 2][2], 0) for k in range(F)]

    dev = lambda a: torch.from_numpy(np.ascontiguousarray(a).view(np.uint8).reshape(-1).copy()).cuda()
    d_pristine, d_blocks = dev(blocks), dev(blocks)
    d_frames = torch.zeros(F * fbytes, dtype=torch.uint8, device="cuda")
    d_qmats, d_qidx, d_off = dev(qmats), dev(qidx), dev(dst_off)
    d_slices = [dev(s) for s in slices]
    base = d_frames.data_ptr()
    works = []
    for k in range(F):
        w = U.picture_works(fr, src[k % 2][2], base + k * fbytes, lambda _: d_blocks.data_ptr() + k * nb * 128, lambda _: d_slices[k].data_ptr())
        works += w
    arr = (tables.FFProresPictureWork * F)(*works)
    h = F // 2
    arr_lo = (tables.FFProresPictureWork * h)(*works[:h])
    arr_hi = (tables.FFProresPictureWork * (F - h))(*works[h:])
    n8 = h * nb
    blocks_of = {"picture": n, "picture_2x8": n, "picture8": n8, "batch8": n8, "batch": n, "idct10": n}
    stride = fr.ls[0]

    def launch(arm):
        if arm == "picture":
            rc = lib.ff_prores_decode_pictures_cuda(arr, F, stream)
        elif arm == "picture_2x8":
            rc = lib.ff_prores_decode_pictures_cuda(arr_lo, h, stream) or lib.ff_prores_decode_pictures_cuda(arr_hi, F - h, stream)
        elif arm == "picture8":
            rc = lib.ff_prores_decode_pictures_cuda(arr_lo, h, stream)
        elif arm in ("batch", "batch8"):
            rc = lib.ff_prores_idct_put_batch_cuda(d_blocks.data_ptr(), base, d_off.data_ptr(), stride, d_qmats.data_ptr(), d_qidx.data_ptr(),
                                                   n if arm == "batch" else n8, stream)
        else:
            rc = lib.ff_simple_idct10_batch_cuda(0, d_blocks.data_ptr(), base, d_off.data_ptr(), stride, n, stream)
        L.check(rc, arm)

    def step(arm):
        d_blocks.copy_(d_pristine)
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        launch(arm)
        e1.record()
        torch.cuda.synchronize()
        return e0.elapsed_time(e1)

    gpu = card()
    for a in ARMS:                      # warm-up
        for _ in range(2):
            step(a)
    times = {a: [] for a in ARMS}
    for _ in range(args.rounds):
        for a in ARMS:
            times[a] += [step(a) for _ in range(args.steps)]
    L.check(0 if not L.last_error() else -1, "timed region")

    # kernel durations from the device trace, one call per arm, in a pass of its own
    from torch.profiler import profile, ProfilerActivity
    kernels = {}
    for a in ARMS:
        d_blocks.copy_(d_pristine)
        torch.cuda.synchronize()
        try:
            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                launch(a)
                torch.cuda.synchronize()
            ks = [(e.time_range.start, e.time_range.end, e.name) for e in prof.events()
                  if ("prores" in e.name or "idct10" in e.name) and e.time_range.end > e.time_range.start]
        except Exception as ex:             # the timing above stands without the trace
            kernels[a] = {"kernels": [], "span_us": None, "gaps_us": [], "error": repr(ex)}
            continue
        ks.sort()
        kernels[a] = {"kernels": [(nm.split("(")[0][-40:], round(t1 - t0, 1)) for t0, t1, nm in ks],
                      "span_us": round(ks[-1][1] - ks[0][0], 1) if ks else None,
                      "gaps_us": [round(ks[j + 1][0] - ks[j][1], 1) for j in range(len(ks) - 1)]}

    # CPU baseline: prores_idct_put_c over the same blocks on every host core
    threads = os.cpu_count() or 1
    hb = blocks.copy()
    hframes = np.zeros(F * fbytes, np.uint8)
    t0 = time.perf_counter()
    assert ref.ref_prores_idct_put_batch(hb.ctypes.data, qmats.ctypes.data, qidx.ctypes.data, hframes.ctypes.data, dst_off.ctypes.data,
                                         stride, n, threads) == 0
    cpu_ms = (time.perf_counter() - t0) * 1e3

    # after the timed region: the picture and batch arms against the reference decoder, every frame
    verified = {}
    for a in ("picture", "batch"):
        d_blocks.copy_(d_pristine)
        d_frames.zero_()
        launch(a)
        torch.cuda.synchronize()
        got = d_frames.cpu().numpy()
        for k in range(F):
            g = got[k * fbytes:(k + 1) * fbytes]
            f0, want = src[k % 2][0], src[k % 2][1]
            if not U.yuv_equal(f0, g, want):
                raise SystemExit("prores_bench.py: arm %s frame %d differs from the reference decoder" % (a, k))
        verified[a] = "y / u / v of all %d frames == reference decoder" % F
    hv = all(U.yuv_equal(src[k % 2][0], hframes[k * fbytes:(k + 1) * fbytes], src[k % 2][1]) for k in range(F))
    verified["cpu"] = "all frames == reference decoder" if hv else "MISMATCH"

    res = {"card": gpu, "frames": F, "blocks": n, "rounds": args.rounds, "steps": args.steps, "verified": verified, "arms": {}, "kernels": kernels,
           "cpu": {"threads": threads, "ms": cpu_ms}}
    print("card (name, power limit, max SM clock): %s" % gpu)
    print("%d frames of %dx%d 4:2:2 HQ per call, %d blocks" % (F, W, H, n))
    print("%-12s %9s %9s %10s %8s %8s" % ("arm", "ms/call", "best", "Gblocks/s", "%HBM", "spread"))
    for a in ARMS:
        tt = sorted(times[a])
        med = tt[len(tt) // 2]
        spread = (tt[-1] - tt[0]) / med
        nb_a = blocks_of[a]
        nbytes = nb_a * (256 if a.startswith("picture") else 384)
        frac = nbytes / (med * 1e-3) / (HBM_TBS * 1e12)
        print("%-12s %9.3f %9.3f %10.2f %7.1f%% %7.2f%%" % (a, med, tt[0], nb_a / (med * 1e-3) / 1e9, 100 * frac, 100 * spread))
        res["arms"][a] = {"blocks": nb_a, "ms_per_call": med, "best_ms": tt[0], "gblocks_per_s": nb_a / (med * 1e-3) / 1e9, "hbm_fraction": frac,
                          "alg_bytes": nbytes, "spread": spread}
    print("cpu      %9.1f ms on %d threads (prores_idct_put_c), %.1fx the picture call" % (cpu_ms, threads, cpu_ms / res["arms"]["picture"]["ms_per_call"]))
    for a in ARMS:
        print("trace %-12s span %s us, kernels (name, us) %s, gaps %s us" % (a, kernels[a]["span_us"], kernels[a]["kernels"], kernels[a]["gaps_us"]))
    print("verified: %s" % verified)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(res, f, indent=1)
    return 0


if __name__ == "__main__":
    sys.exit(main())
