#!/usr/bin/env python
"""sws4k_ceiling.py -- the fused 4K yuv420p->rgb24 kernel set against two ceiling probes, on bench.py's sws4k buffers.

  python tools/sws4k_ceiling.py [--rounds 7] [--steps 1000] [--warmup 50] [--arms kernel,before,move,flat] [--out FILE.json]

Every arm is one setting of the sws_tma_* knobs on the same context and the same two rotating 16-frame buffer sets as bench.py's
sws4k line.  The arms run alternately (A B C A B C ...); each round times `steps` launches with CUDA events after `warmup` untimed
ones.  Printed per arm: the median and the best ms per step over the rounds, the algorithmic rate (1.5 B/px in + 3 B/px out) in TB/s and the
spread (max - min) / median.  Afterwards the scaler's pictures are compared with the CPU checker, as bench.py does.

  before  sws_tma_stages=2 sws_tma_hint=1 sws_tma_pdl=1: the kernel without three stages, L2 hints and dependent launches
  move  sws_tma_probe=1: the kernel's grid, tile order, TMA loads, waits and stores without the arithmetic (wrong pictures)
  flat  sws_tma_probe=2: the same bytes read and written as two linear 16-byte streams (wrong pictures)

The card's name, power limit and maximum SM clock come from a read-only nvidia-smi query and are printed with the numbers.
"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

KNOBS = ("sws_tma_probe", "sws_tma_stages", "sws_tma_hint", "sws_tma_pdl")
# name -> knobs
ARMS = {
    "kernel": {},                                                           # the scaler as bench.py runs it
    "before": {"sws_tma_stages": 2, "sws_tma_hint": 1, "sws_tma_pdl": 1},  # without 3 stages, L2 hints, dependent launches
    "move": {"sws_tma_probe": 1},
    "flat": {"sws_tma_probe": 2},
}


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=30).stdout.strip()
    except Exception as e:          # the numbers still stand; say that the card could not be read
        out = "nvidia-smi unavailable: %s" % e
    return out.splitlines()[0] if out else "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=7)
    ap.add_argument("--steps", type=int, default=1000)
    ap.add_argument("--warmup", type=int, default=50)
    ap.add_argument("--arms", default="kernel,before,move,flat", help="comma-separated arm names")
    ap.add_argument("--out", help="also write the results as JSON to this file")
    args = ap.parse_args()
    names = args.arms.split(",")
    for n in names:
        if n not in ARMS:
            raise SystemExit("unknown arm %r (have: %s)" % (n, ", ".join(ARMS)))

    import torch
    import libav_b200._lib as L
    import bench
    if not torch.cuda.is_available():
        raise SystemExit("sws4k_ceiling.py needs a GPU")
    torch.cuda.set_device(0)
    L.init(0)
    stream = torch.cuda.current_stream().cuda_stream
    wl = bench.make_sws_workload(torch, L, stream, 0)

    def use(arm):
        knobs = ARMS[arm]
        for k in KNOBS:
            L.lib.avb200_set_tuning(k.encode(), int(knobs.get(k, 0)))

    def timed(arm):
        use(arm)
        for i in range(args.warmup):
            wl["run"](i)
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for i in range(args.steps):
            wl["run"](i)
        e1.record()
        torch.cuda.synchronize()
        L.check(0 if not L.last_error() else -1, "sws arm " + arm)
        return e0.elapsed_time(e1) / args.steps

    gpu = card()
    times = {n: [] for n in names}
    for _ in range(args.rounds):
        for n in names:
            times[n].append(timed(n))

    # the scaler's pictures: the last two launches and the host-pointer call, against the CPU checker
    use("kernel")
    wl["run"](0)
    wl["run"](1)
    wl["run_e2e"](0)
    torch.cuda.synchronize()
    verified = wl["verify"]()

    res = {"card": gpu, "rounds": args.rounds, "steps": args.steps, "alg_bytes_per_step": wl["alg_bytes"], "verified": verified, "arms": {}}
    print("card (name, power limit, max SM clock): %s" % gpu)
    print("%-8s %9s %9s %8s %8s" % ("arm", "ms/step", "best", "TB/s", "spread"))
    for n in names:
        t = sorted(times[n])
        med = t[len(t) // 2]
        spread = (t[-1] - t[0]) / med
        tbs = wl["alg_bytes"] / (med * 1e-3) / 1e12
        print("%-8s %9.4f %9.4f %8.3f %7.2f%%" % (n, med, t[0], tbs, 100 * spread))
        res["arms"][n] = {"knobs": ARMS[n], "ms_per_step": med, "tb_per_s": tbs, "spread": spread, "times": times[n]}
    print("verified: %s" % verified)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(res, f, indent=1)
    return 0


if __name__ == "__main__":
    sys.exit(main())
