#!/usr/bin/env python
"""prores_enc_bench.py -- ProRes encoding of sixteen 4096x2160 frames per call (ff_prores_encode_frames_cuda), in three settings:

  hq422      4:2:2, HQ profile, the profile's bit rate
  proxy422   4:2:2, proxy profile, the profile's bit rate
  a4444      4:4:4:4, 4444 profile, 16-bit alpha

  python tools/prores_enc_bench.py [--rounds 5] [--steps 3] [--frames 16] [--out FILE.json]

Source frames are seeded (tests/prores_enc_util.py: smooth gradients, noise and hard edges; two frames, each used for half of the calls'
frames).  The settings alternate within each round; each call is timed alone with CUDA events after a warm-up call per setting, and the
median, best and spread (max - min) / median over rounds x steps are printed with frames/s.  A separate torch.profiler pass (one call per
setting, after the timed region) lists each stage's kernels with their device durations.  The CPU baseline is the reference encoder
(oracle/_ref/libproresencref.so, encode_frame) over the same frames on every host core, one encoder context per thread; after the timed
region every packet of the GPU call is compared with the reference's byte for byte.  The card's name, power limit and maximum SM clock come
from a read-only nvidia-smi query in the same run.  Without a GPU it fails.
"""
import argparse
import ctypes as C
import json
import os
import re
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
sys.path.insert(0, os.path.join(ROOT, "tests"))

W, H = 4096, 2160
SETTINGS = {"hq422": dict(fmt=0, profile=3), "proxy422": dict(fmt=0, profile=0), "a4444": dict(fmt=2, profile=4, alpha_bits=16)}

from xvid_idct_bench import card      # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--frames", type=int, default=16)
    ap.add_argument("--out", help="also write the results as JSON to this file")
    args = ap.parse_args()

    import torch
    import libav_b200._lib as L
    from libav_b200 import tables
    import prores_enc_util as E
    if not torch.cuda.is_available():
        raise SystemExit("prores_enc_bench.py needs a GPU")
    ref = E.ref()
    if ref is None:
        raise SystemExit("prores_enc_bench.py checks with oracle/_ref, which is not built here")
    torch.cuda.set_device(0)
    L.init(0)
    lib = L.lib
    stream = torch.cuda.current_stream().cuda_stream
    F = args.frames

    t0 = time.time()
    setups = {}
    for name, kw in SETTINGS.items():
        src = [E.Case(kw["fmt"], W, H, 0, kw["profile"], 8, alpha_bits=kw.get("alpha_bits", 16), seed=s) for s in (1, 2)]
        planes = [[torch.from_numpy(c.padded(p).reshape(-1).copy()).cuda() if c.planes[p] is not None else None for p in range(4)] for c in src]
        cap = src[0].capacity()
        d_out = torch.zeros(F * cap, dtype=torch.uint8, device="cuda")
        d_size = torch.zeros(F, dtype=torch.int32, device="cuda")
        works = []
        for k in range(F):
            pl = planes[k % 2]
            works.append(src[k % 2].work([p.data_ptr() if p is not None else None for p in pl], d_out.data_ptr() + k * cap, cap,
                                         d_size.data_ptr() + 4 * k))
        arr = (tables.FFProresEncodeWork * F)(*works)
        need = lib.ff_prores_encode_workspace_cuda(arr, F)
        assert need > 0, L.last_error()
        d_ws = torch.empty(need, dtype=torch.uint8, device="cuda")
        setups[name] = dict(src=src, planes=planes, cap=cap, out=d_out, size=d_size, arr=arr, ws=d_ws, need=need)
    print("prepared %d settings in %.1f s" % (len(setups), time.time() - t0))

    def launch(name):
        s = setups[name]
        L.check(lib.ff_prores_encode_frames_cuda(s["arr"], F, s["ws"].data_ptr(), s["need"], stream), name)

    def step(name):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        launch(name)
        e1.record()
        torch.cuda.synchronize()
        return e0.elapsed_time(e1)

    gpu = card()
    for name in SETTINGS:                  # warm-up
        step(name)
    times = {name: [] for name in SETTINGS}
    for _ in range(args.rounds):
        for name in SETTINGS:
            times[name] += [step(name) for _ in range(args.steps)]
    L.check(0 if not L.last_error() else -1, "timed region")

    # kernel durations from the device trace, one call per setting, in a pass of its own
    from torch.profiler import profile, ProfilerActivity
    kernels = {}
    for name in SETTINGS:
        torch.cuda.synchronize()
        try:
            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                launch(name)
                torch.cuda.synchronize()
            ks = [(e.time_range.start, e.time_range.end, e.name) for e in prof.events()
                  if re.search(r"pe_\w+_kernel", e.name) and e.time_range.end > e.time_range.start]
        except Exception as ex:             # the timing above stands without the trace
            kernels[name] = {"stages_us": {}, "error": repr(ex)}
            continue
        stages = {}
        for t_0, t_1, nm in sorted(ks):
            key = re.search(r"pe_\w+_kernel", nm).group(0)
            stages[key] = round(stages.get(key, 0) + t_1 - t_0, 1)
        kernels[name] = {"stages_us": stages, "span_us": round(ks[-1][1] - min(k[0] for k in ks), 1) if ks else None}

    # CPU baseline on every host core, then every GPU packet against the reference's
    threads = os.cpu_count() or 1
    res = {"card": gpu, "frames": F, "size": [W, H], "rounds": args.rounds, "steps": args.steps, "settings": {}, "kernels": kernels}
    print("card (name, power limit, max SM clock): %s" % gpu)
    print("%d frames of %dx%d per call" % (F, W, H))
    print("%-9s %9s %9s %9s %8s %11s %9s" % ("setting", "ms/call", "best", "frames/s", "spread", "cpu ms", "cpu fps"))
    for name in SETTINGS:
        s = setups[name]
        o = s["src"][0].opts()
        hp = [[c.padded(p) for p in range(4)] for c in s["src"]]
        ptrs = (C.c_void_p * (4 * F))(*[hp[k % 2][p].ctypes.data if hp[k % 2][p] is not None else None for k in range(F) for p in range(4)])
        ls = (C.c_int * 4)(*s["src"][0].linesizes())
        houts = [np.zeros(s["cap"], np.uint8) for _ in range(F)]
        optrs = (C.c_void_p * F)(*[h.ctypes.data for h in houts])
        hsizes = np.zeros(F, np.int32)
        t0 = time.perf_counter()
        assert ref.ref_prores_encode_frames(C.byref(o), W, H, F, ptrs, ls, optrs, s["cap"], hsizes.ctypes.data, threads) == 0
        cpu_ms = (time.perf_counter() - t0) * 1e3
        launch(name)
        torch.cuda.synchronize()
        sizes = s["size"].cpu().numpy()
        out = s["out"].cpu().numpy()
        for k in range(F):
            o0, n = k * int(s["cap"]), int(sizes[k])
            if n != int(hsizes[k]) or not np.array_equal(out[o0:o0 + n], houts[k][:n]):
                raise SystemExit("prores_enc_bench.py: %s frame %d differs from the reference encoder's packet" % (name, k))
        tt = sorted(times[name])
        med = tt[len(tt) // 2]
        spread = (tt[-1] - tt[0]) / med
        res["settings"][name] = {"ms_per_call": med, "best_ms": tt[0], "frames_per_s": F / (med * 1e-3), "spread": spread,
                                 "packet_bytes": [int(sizes[0]), int(sizes[1])], "cpu": {"threads": threads, "ms": cpu_ms},
                                 "verified": "all %d packets == reference encoder" % F}
        print("%-9s %9.2f %9.2f %9.1f %7.2f%% %11.1f %9.2f" % (name, med, tt[0], F / (med * 1e-3), 100 * spread, cpu_ms, F / (cpu_ms * 1e-3)))
    for name in SETTINGS:
        print("trace %-9s %s" % (name, kernels[name]))
    print("verified: every packet of every setting == reference encoder (%d frames each)" % F)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(res, f, indent=1)
    return 0


if __name__ == "__main__":
    sys.exit(main())
