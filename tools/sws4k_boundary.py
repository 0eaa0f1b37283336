#!/usr/bin/env python
"""What a launch of the fused 4K yuv420p -> rgb24 kernel costs on top of its frames.

  python tools/sws4k_boundary.py [--lib PATH]... [--rounds 5] [--frames 4096] [--out FILE]

bench.py's sws4k workload (3840x2160, bicubic | accurate_rnd | bitexact, two seeded frames alternating, two buffer sets alternating
between launches), launched back to back with K = 4, 8, 16 and 32 frames per launch and timed with CUDA events.  Per library and round
a least-squares line  ms per launch = a + b * K  is fitted to the four medians: b is the cost of a frame in the steady state, the
intercept a what each launch adds to it -- the start-up and drain at the launch boundary that a longer batch would amortise.
Each --lib is a build of libavdsp_b200.so (default: this tree's); several are timed alternately in every round, so a parent build
and a new one can be compared in one run.  After each timed run the outputs of the last two launches (both buffer sets, every
frame) are compared with the CPU checker's pictures.
"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402

W, H = 3840, 2160
FLAGS = 4 | 0x40000 | 0x80000
KS = (4, 8, 16, 32)


def card():
    """name, power limit and SM clocks of GPU 0 (read-only query)"""
    try:
        r = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                           stdout=subprocess.PIPE, stderr=subprocess.DEVNULL, text=True, timeout=30)
        return r.stdout.strip()
    except (OSError, subprocess.SubprocessError):
        return "nvidia-smi unavailable"


def load(path):
    from libav_b200 import _lib
    lib = C.CDLL(path)
    for name, (res, args) in _lib.PROTOTYPES.items():
        f = getattr(lib, name)
        f.restype, f.argtypes = res, args
    if lib.avb200_init(0) != 0:
        raise SystemExit("%s: avb200_init failed: %s" % (path, lib.avb200_last_error().decode()))
    return lib


def fit(ks, ms):
    b, a = np.polyfit(np.asarray(ks, float), np.asarray(ms, float), 1)
    return a, b


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--lib", action="append", default=[], help="a libavdsp_b200.so build (repeat to alternate builds)")
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--frames", type=int, default=4096, help="frames per timed run (launches = frames / K)")
    ap.add_argument("--warmup", type=int, default=64, help="warm-up frames per run")
    ap.add_argument("--out", help="write the measurements as JSON here")
    args = ap.parse_args()
    libs = args.lib or [os.path.join(ROOT, "libav_b200", "libavdsp_b200.so")]

    import torch
    from libav_b200 import synth
    from oracle import loader
    if not torch.cuda.is_available():
        raise SystemExit("sws4k_boundary.py needs an H100")
    torch.cuda.init()
    builds = [load(os.path.abspath(p)) for p in libs]
    stream = torch.cuda.current_stream()

    kmax = max(KS)
    ysz, csz, osz = W * H, (W // 2) * (H // 2), W * H * 3
    frames = [synth.yuv420p_frame(W, H, 1 + k) for k in range(2)]
    planes = [torch.from_numpy(np.concatenate([frames[k % 2][p].reshape(-1) for k in range(kmax)])) for p in range(3)]
    src = [[p.cuda() for p in planes] for _ in range(2)]
    out = [torch.empty(osz * kmax, dtype=torch.uint8, device="cuda") for _ in range(2)]
    ctxs = []
    for lib in builds:
        ctx = lib.sws_getContext_cuda(W, H, 0, W, H, 2, FLAGS, None, None, None)
        if not ctx or not lib.sws_is_fused_cuda(ctx):
            raise SystemExit("no fused sws4k context")
        ctxs.append(ctx)

    o, kind = (loader.ref(), "reference") if loader.ref() is not None else (loader.port(), "port")
    want = []
    for fr in frames:
        w_ = np.zeros((H, W * 3), np.uint8)
        sp = (C.c_void_p * 3)(*[a.ctypes.data for a in fr]); ss = (C.c_int * 3)(W, W // 2, W // 2)
        if o.sws_yuv420p_to_rgb24(sp, ss, W, H, loader.ptr(w_), W * 3, W, H, FLAGS) != H:
            raise SystemExit("the CPU checker refused the frame")
        want.append(torch.from_numpy(w_).cuda())

    sst = (C.c_int * 3)(W, W // 2, W // 2)
    sf = (C.c_size_t * 3)(ysz, csz, csz)
    dstr = (C.c_int * 3)(W * 3, 0, 0)
    df = (C.c_size_t * 3)(osz, 0, 0)
    args_of = [((C.c_void_p * 3)(*[p.data_ptr() for p in src[k]]), (C.c_void_p * 3)(out[k].data_ptr(), None, None)) for k in range(2)]

    def launch(bi, i, K):
        s, d = args_of[i % 2]
        if builds[bi].sws_scale_frames_cuda(ctxs[bi], s, sst, sf, d, dstr, df, K, C.c_void_p(stream.cuda_stream)) < 0:
            raise SystemExit("%s: sws_scale_frames_cuda failed: %s" % (libs[bi], builds[bi].avb200_last_error().decode()))

    def run(bi, K):
        for i in range(max(2, args.warmup // K)):
            launch(bi, i, K)
        n = max(2, args.frames // K)
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(stream)
        for i in range(n):
            launch(bi, i, K)
        e1.record(stream)
        torch.cuda.synchronize()
        ms = e0.elapsed_time(e1) / n
        for k in range(2):                       # both buffer sets: the last two launches
            got = out[k][:osz * K].view(K, H, W * 3)
            for j in range(K):
                if not torch.equal(got[j], want[j % 2]):
                    raise SystemExit("%s: K=%d frame %d of buffer %d differs from the %s checker" % (libs[bi], K, j, k, kind))
            out[k].fill_(0x5A)                   # the next run's outputs must be its own
        torch.cuda.synchronize()
        return ms

    print("card: %s" % card())
    per = [[[] for _ in KS] for _ in builds]     # [build][K] -> ms per launch, one per round
    for r in range(args.rounds):
        order = list(range(len(builds))) if r % 2 == 0 else list(reversed(range(len(builds))))
        for bi in order:
            for ki, K in enumerate(KS):
                per[bi][ki].append(run(bi, K))
    print("card: %s (after the timed runs)" % card())

    report = {"card": card(), "ks": KS, "rounds": args.rounds, "checker": kind, "builds": []}
    for bi, path in enumerate(libs):
        med = [float(np.median(x)) for x in per[bi]]
        fits = [fit(KS, [per[bi][ki][r] for ki in range(len(KS))]) for r in range(args.rounds)]
        a_r, b_r = [f[0] * 1e3 for f in fits], [f[1] * 1e3 for f in fits]
        a, b = fit(KS, med)
        rep = {"lib": path, "ms_per_launch_median": dict(zip(map(str, KS), med)), "a_us": a * 1e3, "b_us_per_frame": b * 1e3,
               "a_us_rounds": a_r, "b_us_rounds": b_r,
               "spread": {str(K): (max(per[bi][ki]) - min(per[bi][ki])) / med[ki] for ki, K in enumerate(KS)}}
        report["builds"].append(rep)
        print("%s\n  ms per launch (median of %d):  %s" % (path, args.rounds, "  ".join("K=%d %.4f" % (K, m) for K, m in zip(KS, med))))
        print("  fit of the medians: a = %.2f us per launch, b = %.3f us per frame (%.4f ms per 16 frames)" % (a * 1e3, b * 1e3, 16 * b))
        print("  a per round: %s us (min %.2f, max %.2f)" % (" ".join("%.2f" % x for x in a_r), min(a_r), max(a_r)))
        if a * 1e3 < 1.0:
            print("  the per-launch cost is under 1 us: the launch boundary is not where the time goes")
    print("verified: every timed output (both buffer sets, every frame, each K and build) == %s checker" % kind)
    if args.out:
        with open(args.out, "w") as f:
            json.dump(report, f, indent=1)
    for lib, ctx in zip(builds, ctxs):
        lib.sws_freeContext_cuda(ctx)
    return 0


if __name__ == "__main__":
    sys.exit(main())
