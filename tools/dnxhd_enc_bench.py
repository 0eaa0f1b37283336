#!/usr/bin/env python
"""dnxhd_enc_bench.py -- VC-3 / DNxHD encoding of sixteen 1920x1080 frames per call (ff_dnxhd_encode_frames_cuda), in four settings:

  1238_fast   8-bit CID 1238, fast rate control (find_qscale + the variance-ordered step)
  1235_fast   10-bit CID 1235, fast rate control
  1238_rd     8-bit CID 1238, mbd=rd (the lambda search over every qscale's bits and SSD)
  1243_il     8-bit interlaced CID 1243, fast rate control, two coding units per frame

  python tools/dnxhd_enc_bench.py [--rounds 5] [--steps 3] [--frames 16] [--out FILE.json]

Source frames are seeded (tests/dnxhd_enc_util.py: gradients, edges and texture; two frames, alternating).  All frames of a call share one
rate-control state, as one encoder context encodes a sequence, so the search's serial chain from field to field is inside the timing.  The
settings alternate within each round; each call is timed alone with CUDA events after a warm-up call per setting, and the median, best and
spread (max - min) / median over rounds x steps are printed with frames/s.  A separate torch.profiler pass (one call per setting, after the
timed region) lists each stage's kernels with their device durations.  The CPU baseline is the reference encoder
(oracle/_ref/libdnxhdencref.so) over the same frames on every host core, one encoder context per thread; after the timed region a GPU call
from a fresh state is compared packet by packet with the reference encoding the same frames through one context.  The card's name, power
limit and maximum SM clock come from a read-only nvidia-smi query in the same run.  Without a GPU it fails.
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

SETTINGS = {"1238_fast": dict(cid=1238), "1235_fast": dict(cid=1235), "1238_rd": dict(cid=1238, mb_decision=2),
            "1243_il": dict(cid=1243)}

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
    import dnxhd_enc_util as E
    if not torch.cuda.is_available():
        raise SystemExit("dnxhd_enc_bench.py needs a GPU")
    ref = E.ref()
    if ref is None:
        raise SystemExit("dnxhd_enc_bench.py checks with oracle/_ref, which is not built here")
    torch.cuda.set_device(0)
    L.init(0)
    lib = L.lib
    stream = torch.cuda.current_stream().cuda_stream
    F = args.frames

    t0 = time.time()
    setups = {}
    for name, kw in SETTINGS.items():
        cid = kw["cid"]
        case = E.Case(cid, ["natural"] * F, mb_decision=kw.get("mb_decision", 0), seed=1)
        for k in range(2, F):
            case.frames[k] = case.frames[k % 2]
        dev = [[torch.from_numpy(p.reshape(-1).copy()).cuda() for p in case.frames[k][0]] for k in range(2)]
        entry = ref.ref_dnxhd_cid_entry(cid)
        size = C.cast(entry, C.POINTER(tables.FFDnxhdCidEntry))[0].frame_size
        d_out = torch.zeros(F * size, dtype=torch.uint8, device="cuda")
        d_info = torch.zeros(2 * F, dtype=torch.int32, device="cuda")
        d_state = torch.tensor([1, 2 << 10], dtype=torch.int32, device="cuda")
        works = []
        for k in range(F):
            w = tables.FFDnxhdEncodeWork()
            for p in range(3):
                w.data[p] = dev[k % 2][p].data_ptr()
                w.linesize[p] = case.frames[0][1][p]
            w.cid_table = entry
            w.interlaced, w.mb_decision, w.qmax = case.interlaced, case.mb_decision, case.qmax
            w.state = d_state.data_ptr()
            w.out, w.out_capacity, w.out_info = d_out.data_ptr() + k * size, size, d_info.data_ptr() + 8 * k
            works.append(w)
        arr = (tables.FFDnxhdEncodeWork * F)(*works)
        need = lib.ff_dnxhd_encode_workspace_cuda(arr, F)
        assert need > 0, L.last_error()
        d_ws = torch.empty(need, dtype=torch.uint8, device="cuda")
        setups[name] = dict(case=case, dev=dev, size=size, out=d_out, info=d_info, state=d_state, arr=arr, ws=d_ws, need=need)
    print("prepared %d settings in %.1f s" % (len(setups), time.time() - t0))

    def launch(name):
        s = setups[name]
        L.check(lib.ff_dnxhd_encode_frames_cuda(s["arr"], F, s["ws"].data_ptr(), s["need"], stream), name)

    def step(name):
        setups[name]["state"].copy_(torch.tensor([1, 2 << 10], dtype=torch.int32))
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

    from torch.profiler import profile, ProfilerActivity
    kernels = {}
    for name in SETTINGS:
        torch.cuda.synchronize()
        try:
            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                launch(name)
                torch.cuda.synchronize()
            ks = [(e.time_range.start, e.time_range.end, e.name) for e in prof.events()
                  if re.search(r"dn_\w+_kernel", e.name) and e.time_range.end > e.time_range.start]
        except Exception as ex:             # the timing above stands without the trace
            kernels[name] = {"stages_us": {}, "error": repr(ex)}
            continue
        stages = {}
        for t_0, t_1, nm in sorted(ks):
            key = re.search(r"dn_\w+_kernel", nm).group(0)
            stages[key] = round(stages.get(key, 0) + t_1 - t_0, 1)
        kernels[name] = {"stages_us": stages, "span_us": round(ks[-1][1] - min(k[0] for k in ks), 1) if ks else None}

    threads = os.cpu_count() or 1
    res = {"card": gpu, "frames": F, "size": [1920, 1080], "rounds": args.rounds, "steps": args.steps, "settings": {}, "kernels": kernels}
    print("card (name, power limit, max SM clock): %s" % gpu)
    print("%d frames of 1920x1080 per call, one rate-control state per call" % F)
    print("%-10s %9s %9s %9s %8s %11s %9s" % ("setting", "ms/call", "best", "frames/s", "spread", "cpu ms", "cpu fps"))
    for name in SETTINGS:
        s = setups[name]
        case = s["case"]
        planes = (C.c_void_p * (3 * F))(*[p.ctypes.data for f, _ in case.frames for p in f])
        lss = (C.c_int * (3 * F))(*[ls for _, l in case.frames for ls in l])
        hout = np.zeros(F * s["size"], np.uint8)
        hrc = np.zeros(4 * F, np.int32)
        t0 = time.perf_counter()
        assert ref.ref_dnxhd_encode_frames(C.byref(case.opts()), F, planes, lss, hout.ctypes.data, hrc.ctypes.data, threads) == 0
        cpu_ms = (time.perf_counter() - t0) * 1e3
        want, wrc = E.ref_encode(ref, case)                      # one context through all frames, as the GPU call's one state
        step(name)
        out = s["out"].cpu().numpy()
        info = s["info"].cpu().numpy().reshape(F, 2)
        for k in range(F):
            got = out[k * s["size"]:(k + 1) * s["size"]] if info[k, 0] > 0 else None
            E.compare(case, k, got, want[k])
        tt = sorted(times[name])
        med = tt[len(tt) // 2]
        spread = (tt[-1] - tt[0]) / med
        res["settings"][name] = {"ms_per_call": med, "best_ms": tt[0], "frames_per_s": F / (med * 1e-3), "spread": spread,
                                 "cpu": {"threads": threads, "ms": cpu_ms, "frames_per_s": F / (cpu_ms * 1e-3)},
                                 "qscale_after": [int(x) for x in wrc[:, 1]],
                                 "verified": "all %d packets == reference encoder through one context" % F}
        print("%-10s %9.2f %9.2f %9.1f %7.2f%% %11.1f %9.2f" % (name, med, tt[0], F / (med * 1e-3), 100 * spread, cpu_ms, F / (cpu_ms * 1e-3)))
    for name in SETTINGS:
        print("trace %-10s %s" % (name, kernels[name]))
    print("verified: every packet of every setting == reference encoder (%d frames each)" % F)
    print(json.dumps({k: {"gpu_fps": round(v["frames_per_s"], 1), "cpu_fps": round(v["cpu"]["frames_per_s"], 2)} for k, v in res["settings"].items()}))
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(res, f, indent=1)
    return 0


if __name__ == "__main__":
    sys.exit(main())
