#!/usr/bin/env python
"""h263_bench.py -- the H.263 deblocking filter over whole pictures (ff_h263_loop_filter_batch_cuda) and a decoder flush that ends with it
(ff_mpv_flush_pictures_cuda), on HBM-resident batches.

  python tools/h263_bench.py [--rounds 7] [--steps 50] [--warmup 5] [--out FILE.json]

Arms (tests/h263_cases.py pictures: random samples, 25 % skipped macroblocks, qscale 1..31, default chroma qscale table):
  lf_16cif   16 pictures of 1408x1152 (16CIF) in one call
  lf_cif     256 pictures of 352x288 (CIF) in one call (16 launches)
  mc_res     16 H.263 half-sample P pictures of 16CIF: motion compensation and the intra / inter residual a decoder records
             (tests/mpv_mc_cases.py decoder_residual, simple IDCT, intra blocks through the fused h263_intra dequantiser)
  flush      the same flush with the loop filter of those pictures appended
  obmc       16 H.263 P pictures of 16CIF with overlapped block motion compensation (tests/mpv_obmc_cases.py, mostly small vectors)
  mc8x8      the same pictures and vectors without OBMC: every record 8X8 with its four vectors
The arms of a batch alternate within each round; a round times `steps` calls with CUDA events after `warmup` untimed ones.  Printed per
arm: the median and best ms per call, the spread (max - min) / median over the rounds, Mpixel/s (luma pixels), and the algorithmic bytes
over the median time as a fraction of the H100 SXM data sheet's 3.35 TB/s.  The loop filter's model is 1.5 B/px read and 1.5 B/px written
(each 4:2:0 sample once each way) plus 5 B per macroblock of mb_type / qscale_table; the kernel's 8 x 8 tiles partition each plane, so
it reads no halo.  The obmc / mc8x8 arms count 384 B written per macroblock, 384 B of prediction read for mc8x8 and five 8x8 luma
predictions per block (1280 B) plus 128 B of chroma for obmc, and the 44- / 52-byte records.  The flush arms count the motion compensation and residual bytes as tools/mpv_mc_bench.py does.  The CPU figure is the
reference's serial driver (ff_h263_loop_filter per macroblock, oracle/_ref/libh263ref.so, portable C) over the same pictures on all host
cores, one picture per thread.  After timing, every picture is restored and filtered once, and compared with the checker (the serial
reference, else the two-pass port).  The card's name, power limit and maximum SM clock come from a read-only nvidia-smi query.
"""
import argparse
import concurrent.futures as cf
import ctypes as C
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
HBM_TBS = 3.35


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=30).stdout.strip()
    except Exception as e:
        out = "nvidia-smi unavailable: %s" % e
    return out.splitlines()[0] if out else "unknown"


def lf_bytes(pics):
    return sum(1.5 * 256 * p.mb_w * p.mb_h * 2 + 5 * p.mb_w * p.mb_h for p in pics)


def time_arms(L, arms, rounds, steps, warmup):
    e0, e1 = L.lib.avb200_event_create(), L.lib.avb200_event_create()
    ms = {a: [] for a in arms}
    for _ in range(rounds):
        for a, call in arms.items():
            for _ in range(warmup):
                call()
            L.lib.avb200_event_record(e0, None)
            for _ in range(steps):
                call()
            L.lib.avb200_event_record(e1, None)
            L.lib.avb200_event_sync(e1)
            ms[a].append(L.lib.avb200_event_elapsed_ms(e0, e1) / steps)
    L.lib.avb200_event_destroy(e0)
    L.lib.avb200_event_destroy(e1)
    return ms


def summary(ms, nbytes, pixels):
    med = float(np.median(ms))
    return {"ms_median": med, "ms_best": float(min(ms)), "spread": (max(ms) - min(ms)) / med, "mpixel_s": pixels / med / 1e3,
            "algo_TB_s": nbytes / med / 1e9, "hbm_fraction": nbytes / med / 1e9 / HBM_TBS}


def show(name, x):
    print("%-9s: %.3f ms median (best %.3f, spread %.1f %%), %.0f Mpixel/s, %.3f TB/s algorithmic = %.1f %% of %.2f TB/s"
          % (name, x["ms_median"], x["ms_best"], 100 * x["spread"], x["mpixel_s"], x["algo_TB_s"], 100 * x["hbm_fraction"], HBM_TBS))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=7)
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--out")
    args = ap.parse_args()
    import libav_b200._lib as L
    from libav_b200 import device, tables
    from oracle import loader
    import h263_cases as H
    import mpv_mc_cases as M
    L.init(0)
    ref, checker = H.ref_lib(), H.checker_lib()
    results = {"card": card()}
    print("card: %s" % results["card"])

    # ---- the loop filter alone
    batches = {"lf_16cif": (16, 88, 72), "lf_cif": (256, 22, 18)}
    lf = {}
    for name, (n, w, h) in batches.items():
        rng = np.random.default_rng(len(name))
        pics = [H.LfPicture(rng, w, h, skip=0.25, extra_cols=64) for _ in range(n)]
        lf[name] = (pics, H.GpuLf(pics))
    arms = {name: (lambda g=g, n=len(pics): L.check(L.lib.ff_h263_loop_filter_batch_cuda(C.cast(g.arr, C.c_void_p), n, None), "lf"))
            for name, (pics, g) in lf.items()}
    ms = time_arms(L, arms, args.rounds, args.steps, args.warmup)
    for name, (pics, g) in lf.items():
        r = summary(ms[name], lf_bytes(pics), sum(256 * p.mb_w * p.mb_h for p in pics))
        r["pictures"] = len(pics)
        if ref is not None:
            t0 = time.perf_counter()
            with cf.ThreadPoolExecutor(os.cpu_count()) as ex:
                list(ex.map(lambda p: H.run_serial(ref, p), pics))
            r["cpu_ms"], r["cpu_threads"] = (time.perf_counter() - t0) * 1e3, os.cpu_count()
        for fr, pic in zip(g.frames, pics):
            for b, a in zip(fr, pic.bufs):
                L.check(L.lib.avb200_memcpy_h2d(b.ptr, a.ctypes.data, a.nbytes, None), "h2d")
        arms[name]()
        device.sync()
        got = g.download()
        bad = [i for i in range(len(pics)) if H.first_diff(got[i], H.run_serial(checker, pics[i]))]
        r["verified"] = not bad
        results[name] = r
        show(name, r)
        print("%-9s: %d pictures; CPU serial reference %s; verified %s" % (name, len(pics), "%.1f ms on %d threads" % (r["cpu_ms"], r["cpu_threads"])
                                                                          if "cpu_ms" in r else "not available", r["verified"]))

    # ---- a decoder flush with and without the loop filter
    mchk = loader.ref() or loader.port()
    pics = []
    for i in range(16):
        rng = np.random.default_rng(300 + i)
        pic = M.Picture(rng, 2, 88, 72, no_rnd=i & 1)
        M.make_records(rng, pic, far=0.0, edge=0.02)
        pics.append(pic)
    residual = M.decoder_residual(mchk, pics, np.random.default_rng(8), xvid=False, clear=0)
    rng = np.random.default_rng(9)
    tabs = [H.LfPicture(rng, 88, 72, skip=0.25, extra_cols=0) for _ in pics]
    g = M.GpuPictures(pics)
    res = M.GpuResidual(g, residual)
    dev = lambda a: device.DevBuf.from_numpy(np.ascontiguousarray(a))
    keep = [(dev(t.mb_type), dev(t.qscale)) for t in tabs]
    lfa = (tables.FFH263LoopFilterPicture * len(pics))()
    for i, (pic, t) in enumerate(zip(pics, tabs)):
        for k in range(3):
            lfa[i].data[k] = g.frames[i][k].ptr
        lfa[i].linesize, lfa[i].uvlinesize, lfa[i].mb_width, lfa[i].mb_height, lfa[i].mb_stride = pic.p["linesize"], pic.p["uvlinesize"], 88, 72, t.mb_stride
        lfa[i].mb_type, lfa[i].qscale_table = keep[i][0].ptr, keep[i][1].ptr
        lfa[i].chroma_qscale_table[:] = list(range(32))
    w0 = res.work(g)
    w1 = res.work(g)
    w1.loop_filter, w1.n_loop_filter = C.cast(lfa, C.c_void_p), len(pics)
    n_mb_dir = sum(int(((p.recs["mv_dir"] & 1) != 0).sum()) for p in pics)
    mc_bytes = n_mb_dir * 768 + sum(len(p.recs) for p in pics) * 44
    res_bytes = sum(len(b["off"]) * (192 + (64 if b["mode"] == 1 and b["dq"] < 0 else 0) + (4 if b["dq"] >= 0 else 0)) for b in residual)
    arms = {"mc_res": lambda: L.check(L.lib.ff_mpv_flush_pictures_cuda(C.byref(w0), None), "flush"),
            "flush": lambda: L.check(L.lib.ff_mpv_flush_pictures_cuda(C.byref(w1), None), "flush")}
    ms = time_arms(L, arms, args.rounds, args.steps, args.warmup)
    pixels = sum(256 * 88 * 72 for _ in pics)
    results["mc_res"] = summary(ms["mc_res"], mc_bytes + res_bytes, pixels)
    results["flush"] = summary(ms["flush"], mc_bytes + res_bytes + lf_bytes(tabs), pixels)
    want = [M.run_ref(M.checker_lib(), p) for p in pics]
    M.apply_residual(mchk, M.xvid_checker(), want, residual)
    for pic, wnt, t in zip(pics, want, tabs):
        prm = np.array([pic.p["linesize"], pic.p["uvlinesize"], 88, 72, t.mb_stride], np.int32)
        ct = np.arange(32, dtype=np.uint8)
        assert checker.picture((C.c_void_p * 3)(*[a.ctypes.data for a in wnt]), prm.ctypes.data, t.mb_type.ctypes.data, t.qscale.ctypes.data,
                               ct.ctypes.data) == 0
    for fr, pic in zip(g.frames, pics):
        for b, a in zip(fr, pic.frame):
            L.check(L.lib.avb200_memcpy_h2d(b.ptr, a.ctypes.data, a.nbytes, None), "h2d")
    arms["flush"]()
    device.sync()
    got = g.download()
    results["flush"]["verified"] = not [i for i in range(len(pics)) if M.first_diff(got[i], want[i])] and g.rejected() == 0
    show("mc_res", results["mc_res"])
    show("flush", results["flush"])
    print("flush: 16 x 16CIF H.263 P pictures, %d residual batches; loop filter share of the flush %.3f ms; verified %s"
          % (len(residual), results["flush"]["ms_median"] - results["mc_res"]["ms_median"], results["flush"]["verified"]))
    # ---- OBMC against plain 4MV motion compensation, same pictures and vectors
    import mpv_obmc_cases as O
    pics = [O.obmc_picture(np.random.default_rng(500 + i), 88, 72, no_rnd=i & 1, far=0.0, edge=0.02, stale=0.0, intra=0.05) for i in range(16)]
    for p in pics:
        p.recs["mv_type"] = M.T8X8
        p.recs["mv"][:, 0] = p.obmc["mv"]
    gs = {}
    for name, on in (("obmc", 1), ("mc8x8", 0)):
        g = M.GpuPictures(pics)
        obs = [device.DevBuf.from_numpy(np.ascontiguousarray(p.obmc)) for p in pics]
        for i in range(len(pics)):
            g.arr[i].obmc, g.arr[i].obmc_recs = on, obs[i].ptr
        gs[name] = (g, obs)
    arms = {name: (lambda g=g: L.check(L.lib.ff_mpv_motion_batch_cuda(C.cast(g.arr, C.c_void_p), len(pics), g.rej.ptr, None), name))
            for name, (g, _) in gs.items()}
    ms = time_arms(L, arms, args.rounds, args.steps, args.warmup)
    n_rec = sum(len(p.recs) for p in pics)
    pixels = 16 * 256 * 88 * 72
    results["obmc"] = summary(ms["obmc"], n_rec * (384 + 1280 + 128 + 44 + 52), pixels)
    results["mc8x8"] = summary(ms["mc8x8"], n_rec * (384 + 384 + 44), pixels)
    ob_check = O.checker_lib()
    for name, (g, _) in gs.items():
        for fr, pic in zip(g.frames, pics):
            for b, a in zip(fr, pic.frame):
                L.check(L.lib.avb200_memcpy_h2d(b.ptr, a.ctypes.data, a.nbytes, None), "h2d")
        arms[name]()
        device.sync()
        got = g.download()
        ref = (lambda p: O.run_ref(ob_check, p)) if name == "obmc" else (lambda p: M.run_ref(M.checker_lib(), p))
        results[name]["verified"] = not [i for i in range(len(pics)) if M.first_diff(got[i], ref(pics[i]))] and g.rejected() == 0
        show(name, results[name])
    print("obmc / mc8x8: 16 x 16CIF P pictures, %d records; verified %s / %s" % (n_rec, results["obmc"]["verified"], results["mc8x8"]["verified"]))
    if args.out:
        with open(args.out, "w") as f:
            json.dump(results, f, indent=1)


if __name__ == "__main__":
    main()
