#!/usr/bin/env python
"""dnxhd_dec_bench.py -- VC-3 / DNxHD decoding (ff_dnxhd_decode_frames_cuda) of 1920x1080 packets, 1, 16 and 64 per call, in four settings:

  1238   8-bit CID 1238 (the reference encoder's packets)
  1235   10-bit CID 1235
  1243   8-bit interlaced CID 1243, two coding units per packet
  1256   10-bit 4:4:4 CID 1256 (synthesised: the reference encoder does not write 4:4:4)

  python tools/dnxhd_dec_bench.py [--steps 10] [--out FILE.json]

Packets are seeded (tests/dnxhd_dec_util.py; two per setting, alternating).  Device-resident: packets and planes stay on the device, each
call is timed with CUDA events after a warm-up call, median over steps.  End to end: packet upload, the call and the download of the
frames, on a host clock around work that ends in a synchronise.  A separate torch.profiler pass, one session over a 64-packet call per
setting, lists the two stages' kernels with their device durations.  The CPU baseline is the reference decoder (oracle/_ref/libdnxhddecref.so: the portable C build,
without the x86 SIMD IDCT, with the checked bitstream reader) over the same packets on every host core, one context per thread.  After the timed region every frame of one 64-packet call per setting is compared
byte for byte with the reference decoder.  The card's name, power limit and maximum SM clock come from a read-only nvidia-smi query in the
same run.  Without a GPU it fails.
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


def packets(dref, eref, name):
    import dnxhd_dec_util as D
    if name == "1256":
        return [D.synth(dref, D.Synth(1256, seed=k, is444=True, eob=0.08, qscales=(2, 4, 8))) for k in range(2)]
    return D.real_packets(eref, int(name), ["natural", "noise"], seed=5)


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
    lib, dref, eref = L.lib, D.ref(), E.ref()
    cids, ncids, _ = D.cid_table(dref)
    gpu = card()
    print("card (name, power limit, max SM clock): %s" % gpu)
    dev = torch.device("cuda")
    results = {"card": gpu, "settings": {}}
    threads = os.cpu_count()
    prof_calls = []
    for name in ("1238", "1235", "1243", "1256"):
        pk = packets(dref, eref, name)
        ret, info = D.info_of(lib, pk[0], cids, ncids)
        assert ret == 0
        bpp = 1 if info.pix_fmt == 4 else 2
        cw = info.width if info.pix_fmt == 70 else info.width // 2
        lss = [info.width * bpp, cw * bpp, cw * bpp]
        res = {}
        for n in (1, 16, 64):
            host = [np.frombuffer(pk[k % 2], np.uint8).copy() for k in range(n)]
            dpk = [torch.from_numpy(h).to(dev) for h in host]
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
            st = torch.cuda.current_stream().cuda_stream

            def call(arr=arr, n=n, ws=ws, need=need, st=st, keep=(host, dpk, planes)):   # bound now: the profiler pass calls it later
                assert lib.ff_dnxhd_decode_frames_cuda(arr, n, cids, ncids, C.c_void_p(ws.data_ptr()), need, C.c_void_p(st)) == 0
            call(); torch.cuda.synchronize()
            ts = []
            for _ in range(a.steps):
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record(); call(); e1.record(); e1.synchronize()
                ts.append(e0.elapsed_time(e1))
            pinned = [torch.from_numpy(h).pin_memory() for h in host]
            outs = [[torch.empty((info.lines, ls), dtype=torch.uint8).pin_memory() for ls in lss] for _ in range(n)]
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            for _ in range(a.steps):
                for k in range(n):
                    dpk[k].copy_(pinned[k], non_blocking=True)
                call()
                for k in range(n):
                    for p in range(3):
                        outs[k][p].copy_(planes[k][p], non_blocking=True)
                torch.cuda.synchronize()
            e2e = (time.perf_counter() - t0) / a.steps
            res[n] = {"device_ms_per_call": float(np.median(ts)), "device_frames_per_s": n / (np.median(ts) / 1e3),
                      "e2e_frames_per_s": n / e2e, "spread": float((max(ts) - min(ts)) / np.median(ts))}
            print("%s n=%2d  device %.3f ms/call (%.0f frames/s, spread %.2f)  with upload+download %.0f frames/s" % (
                name, n, res[n]["device_ms_per_call"], res[n]["device_frames_per_s"], res[n]["spread"], res[n]["e2e_frames_per_s"]))
        # reference on every host core
        nref = 64
        refp = [[np.full((max(info.lines, info.height), ls), D.SENTINEL, np.uint8) for ls in lss] for _ in range(nref)]
        pkts = [np.frombuffer(pk[k % 2], np.uint8).copy() for k in range(nref)]
        pp = (C.c_void_p * nref)(*[p.ctypes.data for p in pkts])
        sz = (C.c_int * nref)(*[len(p) for p in pkts])
        pl = (C.c_void_p * (3 * nref))(*[x.ctypes.data for f in refp for x in f])
        ls3 = (C.c_int * (3 * nref))(*(lss * nref))
        t0 = time.perf_counter()
        dref.ref_dnxhd_decode_frames(pp, sz, nref, pl, ls3, max(info.lines, info.height), threads)
        tref = time.perf_counter() - t0
        res["reference_frames_per_s"] = nref / tref
        res["reference_threads"] = threads
        print("%s reference decoder, %d host threads: %.1f frames/s" % (name, threads, nref / tref))
        prof_calls.append((name, call))
        # correctness after the timed region: the last 64-packet call, frame by frame
        torch.cuda.synchronize()
        for k in range(64):
            _, want, _, _ = D.ref_decode(dref, pk[k % 2], info)
            for p in range(3):
                got = planes[k][p].cpu().numpy()
                assert np.array_equal(got, want[p][:info.lines]), ("mismatch", name, k, p)
        print("%s: all 64 frames equal the reference decoder's" % name)
        results["settings"][name] = res
    # per-stage kernel time: one profiler session over one 64-packet call per setting, in order.  A call is one entropy launch followed by
    # one put launch per field, so the kernels, sorted by start, split into calls at each entropy launch.
    from torch.profiler import profile, ProfilerActivity
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _, call in prof_calls:
            call()
            torch.cuda.synchronize()
    kernels = sorted(((ev.time_range.start, ev.name, ev.time_range.elapsed_us()) for ev in prof.events()
                      if ev.device_type == torch.autograd.DeviceType.CUDA and ("dd_entropy_kernel" in ev.name or "dd_put_kernel" in ev.name)))
    calls = []
    for _, kname, us in kernels:
        if "dd_entropy_kernel" in kname:
            calls.append({})
        stage = "entropy" if "dd_entropy_kernel" in kname else "put"
        calls[-1][stage] = calls[-1].get(stage, 0.0) + us / 1e3
    assert len(calls) == len(prof_calls), ("profiler kernels", [k[1][:60] for k in kernels])
    for (name, _), st in zip(prof_calls, calls):
        results["settings"][name]["stages_ms_64"] = st
        print("%s stages at 64 packets (ms): %s" % (name, ", ".join("%s %.3f" % kv for kv in st.items())))
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        json.dump(results, open(a.out, "w"), indent=1, default=str)


if __name__ == "__main__":
    main()
