#!/usr/bin/env python
"""prores_dec_bench.py -- ProRes decoding (ff_prores_decode_frames_cuda), 1, 16 and 64 packets per call, at 1920x1080 and 4096x2160, in
the ProRes encoder bench's settings:

  hq        4:2:2 HQ
  proxy     4:2:2 proxy
  4444      4:4:4:4 with 16-bit alpha
  hq_tff    4:2:2 HQ, interlaced, top field first

  python tools/prores_dec_bench.py [--steps 5] [--sizes 1920x1080,4096x2160] [--sweep] [--out FILE.json]

Packets come from the reference encoder (tests/prores_dec_util.py; two seeds per setting, alternating).  Device-resident: packets and planes
stay on the device, each call is timed with CUDA events after a warm-up call, median over steps.  End to end: packet upload, the call and
the download of the frames, on a host clock around work that ends in a synchronise.  A torch.profiler pass over one 64-packet call per
setting lists each stage's kernels with their device durations.  The CPU column is the reference decoder (oracle/_ref/libproresdecref.so:
the portable C build with the checked bitstream reader) over the same packets on every host core, one fresh context per packet.  After the
timed region the first 16 frames of one 64-packet call per setting are compared byte for byte with the reference decoder.  --sweep times the
entropy stage's active lanes per warp (the prd_lanes test knob) at 16 and 64 packets, and the alpha stage's (prd_alpha_lanes) for 4444;
the compared call runs after the sweep, with the shipped shapes.  The card's name, power limit and maximum SM clock come from a read-only
nvidia-smi query in the same run.  Without a GPU it fails.
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

from xvid_idct_bench import card      # noqa: E402

SETTINGS = {"hq": (0, 0, 3), "proxy": (0, 0, 0), "4444": (2, 0, 4), "hq_tff": (0, 1, 3)}     # fmt, interlaced, profile
STAGES = (("prd_chunk_kernel", "offsets"), ("prd_offset_kernel", "offsets"), ("prd_entropy_kernel", "entropy"),
          ("prd_alpha_kernel", "alpha"), ("prores_picture", "put"))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--sizes", default="1920x1080,4096x2160")
    ap.add_argument("--sweep", action="store_true")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import torch
    assert torch.cuda.is_available(), "needs a GPU"
    import __graft_entry__ as g
    g.build()
    import libav_b200._lib as L
    L.init(0)
    import prores_dec_util as D
    import prores_enc_util as E
    from libav_b200 import tables
    lib, dref, eref = L.lib, D.ref(), E.ref()
    gpu = card()
    print("card (name, power limit, max SM clock): %s" % gpu)
    dev = torch.device("cuda")
    results = {"card": gpu, "settings": {}, "sweep": {}}
    threads = os.cpu_count()
    prof_calls = []
    for size in a.sizes.split(","):
        W, H = map(int, size.split("x"))
        for name, (fmt, il, prof) in SETTINGS.items():
            key = "%s_%s" % (name, size)
            pk = [D.encode(eref, fmt, W, H, interlaced=il, profile=prof, seed=s) for s in (1, 2)]
            ret, info = D.probe(lib, pk[0])
            assert ret == 0
            ls = 32 * ((W + 15) // 16)
            res = {"packet_bytes": [len(p.data) for p in pk]}
            calls = {}
            for n in (1, 16, 64):
                host = [np.frombuffer(pk[k % 2].data, np.uint8).copy() for k in range(n)]
                dpk = [torch.from_numpy(h).to(dev) for h in host]
                planes = [[torch.full((info.lines, ls), D.SENTINEL, dtype=torch.uint8, device=dev) for _ in range(4)] for _ in range(n)]
                works = []
                for k in range(n):
                    w = tables.FFProresDecodeWork(pkt_host=host[k].ctypes.data, pkt=dpk[k].data_ptr(), size=len(host[k]), width=W, height=H)
                    for p in range(4):
                        w.data[p], w.linesize[p], w.lines[p] = planes[k][p].data_ptr(), ls, info.lines
                    works.append(w)
                arr = (tables.FFProresDecodeWork * n)(*works)
                need = lib.ff_prores_decode_workspace_cuda(arr, n)
                ws = torch.empty(need, dtype=torch.uint8, device=dev)
                st = torch.cuda.current_stream().cuda_stream

                def call(arr=arr, n=n, ws=ws, need=need, st=st, keep=(host, dpk, planes)):   # bound now: the profiler pass calls it later
                    assert lib.ff_prores_decode_frames_cuda(arr, n, C.c_void_p(ws.data_ptr()), need, C.c_void_p(st)) == 0

                def timed(steps):
                    call(); torch.cuda.synchronize()
                    ts = []
                    for _ in range(steps):
                        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                        e0.record(); call(); e1.record(); e1.synchronize()
                        ts.append(e0.elapsed_time(e1))
                    return ts
                ts = timed(a.steps)
                nplanes = 4 if fmt == 2 else 3
                pinned = [torch.from_numpy(h).pin_memory() for h in host]
                outs = [[torch.empty((info.lines, ls), dtype=torch.uint8).pin_memory() for _ in range(nplanes)] for _ in range(n)]
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                for _ in range(a.steps):
                    for k in range(n):
                        dpk[k].copy_(pinned[k], non_blocking=True)
                    call()
                    for k in range(n):
                        for p in range(nplanes):
                            outs[k][p].copy_(planes[k][p], non_blocking=True)
                    torch.cuda.synchronize()
                e2e = (time.perf_counter() - t0) / a.steps
                med = float(np.median(ts))
                res[n] = {"device_ms_per_call": med, "device_frames_per_s": n / (med / 1e3), "e2e_frames_per_s": n / e2e,
                          "spread": float((max(ts) - min(ts)) / med)}
                print("%s n=%2d  device %.3f ms/call (%.0f frames/s, spread %.2f)  with upload+download %.0f frames/s" % (
                    key, n, med, res[n]["device_frames_per_s"], res[n]["spread"], res[n]["e2e_frames_per_s"]))
                if a.sweep and n in (16, 64) and name in ("hq", "4444"):
                    sw = {}
                    for lanes in (1, 2, 4, 8, 16, 32):
                        lib.avb200_set_tuning(b"prd_lanes", lanes)
                        sw[lanes] = float(np.median(timed(a.steps)))
                    lib.avb200_set_tuning(b"prd_lanes", 0)
                    results["sweep"]["%s_n%d" % (key, n)] = sw
                    print("%s n=%d lanes sweep (ms/call): %s" % (key, n, ", ".join("%d: %.3f" % kv for kv in sw.items())))
                    if fmt == 2:
                        sw = {}
                        for lanes in (1, 2, 4, 8, 16, 32):
                            lib.avb200_set_tuning(b"prd_alpha_lanes", lanes)
                            sw[lanes] = float(np.median(timed(a.steps)))
                        lib.avb200_set_tuning(b"prd_alpha_lanes", 0)
                        results["sweep"]["%s_n%d_alpha" % (key, n)] = sw
                        print("%s n=%d alpha lanes sweep (ms/call): %s" % (key, n, ", ".join("%d: %.3f" % kv for kv in sw.items())))
                calls[n] = (call, planes)
            # the reference decoder on every host core, over the first 16 packets of the 64-packet call
            nref = 16
            refp = [[np.full((info.lines, ls), D.SENTINEL, np.uint8) for _ in range(4)] for _ in range(nref)]
            pkts = [np.frombuffer(pk[k % 2].data, np.uint8).copy() for k in range(nref)]
            pp = (C.c_void_p * nref)(*[p.ctypes.data for p in pkts])
            sz = (C.c_int * nref)(*[len(p) for p in pkts])
            pl = (C.c_void_p * (4 * nref))(*[x.ctypes.data for f in refp for x in f])
            ls4 = (C.c_int * (4 * nref))(*([ls] * 4 * nref))
            t0 = time.perf_counter()
            dref.ref_prores_dec_decode_frames(pp, sz, nref, W, H, pl, ls4, threads)
            tref = time.perf_counter() - t0
            res["reference_frames_per_s"] = nref / tref
            res["reference_threads"] = threads
            print("%s reference decoder (portable C, checked reader), %d host threads: %.1f frames/s" % (key, threads, nref / tref))
            # correctness after the timed region: the 64-packet call's first 16 frames (both packets), byte for byte
            torch.cuda.synchronize()
            calls[64][0]()                                           # the shipped launch shapes, after any sweep
            torch.cuda.synchronize()
            planes = calls[64][1]
            for k in range(nref):
                want = refp[k]
                for p in range(4):
                    got = planes[k][p].cpu().numpy()
                    assert np.array_equal(got, want[p]), ("mismatch", key, k, p)
            print("%s: the 64-packet call's first %d frames equal the reference decoder's" % (key, nref))
            prof_calls.append((key, calls[64][0]))
            results["settings"][key] = res
    # per-stage kernel time: one profiler session, one 64-packet call per setting in order, each call bracketed by a synchronise; a call's
    # kernels start at its first chunk kernel
    from torch.profiler import profile, ProfilerActivity
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _, call in prof_calls:
            call()
            torch.cuda.synchronize()
    kernels = sorted((ev.time_range.start, ev.name, ev.time_range.elapsed_us()) for ev in prof.events()
                     if ev.device_type == torch.autograd.DeviceType.CUDA and any(s in ev.name for s, _ in STAGES))
    per_call = []
    for _, kname, us in kernels:
        if "prd_chunk_kernel" in kname:
            per_call.append({})
        stage = next(label for s, label in STAGES if s in kname)
        per_call[-1][stage] = per_call[-1].get(stage, 0.0) + us / 1e3
    assert len(per_call) == len(prof_calls), ("profiler kernels", len(per_call), len(prof_calls))
    for (key, _), stt in zip(prof_calls, per_call):
        results["settings"][key]["stages_ms_64"] = stt
        print("%s stages at 64 packets (ms): %s" % (key, ", ".join("%s %.3f" % kv for kv in stt.items())))
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        json.dump(results, open(a.out, "w"), indent=1, default=str)


if __name__ == "__main__":
    main()
