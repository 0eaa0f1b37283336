#!/usr/bin/env python
"""mpv_mc_bench.py -- batched mpegvideo motion compensation (ff_mpv_motion_batch_cuda) and the whole flush (ff_mpv_flush_pictures_cuda:
motion compensation, then the residual batches) on HBM-resident batches.

  python tools/mpv_mc_bench.py [--rounds 7] [--steps 50] [--warmup 5] [--out FILE.json]

Five batches of sixteen 1920x1088 pictures, records generated with mostly small vectors (tests/mpv_mc_cases.py); 8 % of the macroblocks are
intra (no MC, six coded blocks), each block of an inter macroblock is coded at probability 0.5 (tests/mpv_mc_cases.py decoder_residual):
  mpeg2  MPEG-2: frame P and B pictures (16X16, FIELD, DMV; half the macroblocks with field DCT) and field pictures (FIELD, 16X8, DMV),
         first and second fields; simple IDCT, idct_put for intra and idct_add for inter blocks
  mpeg4  MPEG-4 ASP as Xvid writes it: quarter-sample P and B pictures, 16X16 and 4MV, bi-predicted 8x8 records like B-direct; the Xvid
         IDCT, intra blocks through the fused h263_intra dequantiser, inter blocks added
  mpeg4_gmc  MPEG-4 ASP S-VOPs with GMC (tests/mpv_gmc_cases.py): 2- and 3-point warps from random sprite trajectories, about 70 % of the
         macroblocks mcsel 16X16 (four in five of them skipped: no residual), the rest quarter-sample 16X16 and 4MV; residual as mpeg4
  mpeg2_422  MPEG-2 4:2:2 (tests/mpv_ilace_cases.py), mixed like mpeg2; eight blocks per macroblock, field DCT in frame pictures moving
         the chroma blocks too
  mpeg4_ilace  interlaced MPEG-4 ASP: P and B pictures, quarter- and half-sample, about half of the macroblocks FIELD records (B-direct
         ones among them), the rest 16X16 and 4MV; the Xvid IDCT with field DCT in half of the macroblocks
The residual batches run without `clear`, so every timed flush transforms the same coefficients.  The arms `mc` (the motion compensation
alone) and `flush` alternate within each round; a round times `steps` calls with CUDA events after `warmup` untimed ones.  Printed per
batch and arm: the median and best ms per call, the spread (max - min) / median over the rounds, Mpixel/s of predicted pictures, and the
algorithmic bytes over the median time as a fraction of the H100 SXM data sheet's 3.35 TB/s.  Bytes: per macroblock and direction 384 B
of prediction read and 384 B written (4:2:2: 512 B each), plus the 44-byte record; per residual block 128 B of coefficients read and 64 B of pixels written
(+ 64 B read for add, + 4 B of dequantiser record).  The CPU figure is the reference's own ff_mpv_motion (oracle/_ref/libmpvmcref.so,
portable C; ref_mpvmc_gmc_picture of oracle/_ref/libmpvgmcref.so for the S-VOPs, ref_mpvmc_cf_picture of libmpvcfref.so for 4:2:2) over the same records on all host cores, one picture per thread (motion compensation
only).  After timing, every picture is
rebuilt from its original bytes by one flush and compared with the chained checker: the reference's MC, then the IDCT and inverse
quantiser oracles over the same batches.  The card's name, power limit and maximum SM clock come from a read-only nvidia-smi query and are
printed with the numbers.
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


def gmc_batch(checker):
    """sixteen S-VOPs; the residual of skipped mcsel macroblocks is dropped"""
    import mpv_gmc_cases as G
    import mpv_mc_cases as M
    pics, skipped = [], []
    for i in range(16):
        rng = np.random.default_rng(2000 + i)
        pic = M.Picture(rng, 2, 120, 68, no_rnd=(i >> 1) & 1, qpel=1, width=1920, height=1080)
        old = M.make_records(rng, pic, far=0.0, edge=0.02, types=[M.T16X16, M.T8X8])
        recs = np.zeros(len(old), G.REC)
        for name in M.REC.names:
            if name != "pad":
                recs[name] = old[name]
        recs["mv_dir"] = 1
        recs["mcsel"] = rng.random(len(recs)) < 0.7
        recs["mv_type"][recs["mcsel"] == 1] = M.T16X16
        pic.recs = recs
        pic.sprite = G.random_params(rng, 1920, 1080, 120, 68, 1920, 1080, pts=2 + (i & 1), scale=16)
        skipped.append({(int(r["mb_x"]), int(r["mb_y"])) for r in recs if r["mcsel"] and rng.random() < 0.8})
        pics.append(pic)
    residual = M.decoder_residual(checker, pics, np.random.default_rng(9), xvid=True, clear=0)
    for b in residual:
        if b["dq"] >= 0:
            continue                                         # intra blocks
        pic = pics[b["pi"]]
        ls = pic.p["linesize"] if b["pl"] == 0 else pic.p["uvlinesize"]
        mb = 16 if b["pl"] == 0 else 8
        keep = np.array([((int(o) % ls) // mb, (int(o) // ls) // mb) not in skipped[b["pi"]] for o in b["off"]], bool)
        b["off"], b["blocks"], b["rec"] = np.ascontiguousarray(b["off"][keep]), np.ascontiguousarray(b["blocks"][keep]), b["rec"][keep]
    return pics, [b for b in residual if len(b["off"])]


def ilace_batch(kind, checker):
    """sixteen MPEG-2 4:2:2 pictures or sixteen interlaced MPEG-4 pictures, with a decoder's residual"""
    import mpv_ilace_cases as I
    import mpv_mc_cases as M
    pics = []
    for i in range(16):
        rng = np.random.default_rng(3000 + 100 * (kind == "mpeg4_ilace") + i)
        if kind == "mpeg2_422":
            st, ff, b = [(M.FRAME, 1, 0), (M.FRAME, 1, 1), (M.TOP, 1, 0), (M.BOTTOM, 0, 0)][i % 4]
            pics.append(I.cf_picture(rng, 2, 120, 68, structure=st, first_field=ff, b=b, far=0.0, edge=0.02))
        else:
            pic = I.IlacePicture(rng, 120, 68, b=i & 1, no_rnd=(i >> 2) & 1, qpel=(i >> 1) & 1, width=1920, height=1080)
            I.ilace_records(rng, pic, field=0.5, far=0.0, edge=0.02)
            pics.append(pic)
    return pics, I.residual(checker, pics, np.random.default_rng(11), xvid=kind == "mpeg4_ilace", clear=0)


class _Ilace:
    """the mpeg2_422 / mpeg4_ilace pictures' reference and checker (both the reference itself: tests/mpv_ilace_cases.py)"""

    @staticmethod
    def ref_lib():
        import mpv_ilace_cases as I
        return I.cf_ref_lib() if I.have_reference() else None

    checker_lib = ref_lib

    @staticmethod
    def run_ref(lib, pic):
        import mpv_ilace_cases as I
        return I.run_ref(pic)


def batch(kind, checker):
    import mpv_mc_cases as M
    if kind == "mpeg4_gmc":
        return gmc_batch(checker)
    if kind in ("mpeg2_422", "mpeg4_ilace"):
        return ilace_batch(kind, checker)
    pics = []
    for i in range(16):
        rng = np.random.default_rng(1000 * (kind == "mpeg4") + i)
        if kind == "mpeg2":
            st, ff, b = [(M.FRAME, 1, 0), (M.FRAME, 1, 1), (M.TOP, 1, 0), (M.BOTTOM, 0, 0)][i % 4]
            pic = M.Picture(rng, 0, 120, 68, structure=st, first_field=ff, b=b)
        else:
            pic = M.Picture(rng, 2, 120, 68, b=i & 1, no_rnd=(i >> 1) & 1, qpel=1, width=1920, height=1080)
        M.make_records(rng, pic, far=0.0, edge=0.02)
        pics.append(pic)
    residual = M.decoder_residual(checker, pics, np.random.default_rng(7 + (kind == "mpeg4")), xvid=kind == "mpeg4", clear=0)
    return pics, residual


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=7)
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--out")
    args = ap.parse_args()
    import libav_b200._lib as L
    from libav_b200 import device
    from oracle import loader
    import mpv_gmc_cases as G
    import mpv_ilace_cases as I
    import mpv_mc_cases as M
    L.init(0)
    checker = loader.ref() or loader.port()
    results = {"card": card()}
    print("card: %s" % results["card"])
    for kind in ("mpeg2", "mpeg4", "mpeg4_gmc", "mpeg2_422", "mpeg4_ilace"):
        new_kind = kind in ("mpeg2_422", "mpeg4_ilace")
        C_ = G if kind == "mpeg4_gmc" else _Ilace if new_kind else M          # the pictures' reference and checker
        ref, mc_checker = C_.ref_lib(), C_.checker_lib()
        pics, residual = batch(kind, checker)
        g = G.GpuSvops(pics) if kind == "mpeg4_gmc" else I.GpuPics(pics) if new_kind else M.GpuPictures(pics)
        res = M.GpuResidual(g, residual)
        work = res.work(g)
        n_mb_dir = sum(int(((p.recs["mv_dir"] & 1) != 0).sum() + ((p.recs["mv_dir"] & 2) != 0).sum()) for p in pics)
        n_rec = sum(len(p.recs) for p in pics)
        mc_bytes = n_mb_dir * (1024 if kind == "mpeg2_422" else 768) + n_rec * 44
        res_bytes = sum(len(b["off"]) * (192 + (64 if (b["mode"] == 1 and b["dq"] < 0) or b["dq"] in (1, 4, 6) else 0) + (4 if b["dq"] >= 0 else 0))
                        for b in residual)
        pixels = sum(16 * p.mb_rows * 16 * p.p["mb_width"] for p in pics)
        arms = {
            "mc": (lambda: L.check(L.lib.ff_mpv_motion_batch_cuda(C.cast(g.arr, C.c_void_p), len(pics), g.rej.ptr, None), "mc"), mc_bytes),
            "flush": (lambda: L.check(L.lib.ff_mpv_flush_pictures_cuda(C.byref(work), None), "flush"), mc_bytes + res_bytes),
        }
        e0, e1 = L.lib.avb200_event_create(), L.lib.avb200_event_create()
        ms = {a: [] for a in arms}
        for _ in range(args.rounds):
            for a, (call, _) in arms.items():
                for _ in range(args.warmup):
                    call()
                L.lib.avb200_event_record(e0, None)
                for _ in range(args.steps):
                    call()
                L.lib.avb200_event_record(e1, None)
                L.lib.avb200_event_sync(e1)
                ms[a].append(L.lib.avb200_event_elapsed_ms(e0, e1) / args.steps)
        r = {"records": n_rec, "mb_directions": n_mb_dir, "residual_batches": len(residual), "residual_blocks": sum(len(b["off"]) for b in residual)}
        for a, (_, nbytes) in arms.items():
            med = float(np.median(ms[a]))
            r[a] = {"ms_median": med, "ms_best": float(min(ms[a])), "spread": (max(ms[a]) - min(ms[a])) / med, "mpixel_s": pixels / med / 1e3,
                    "algo_TB_s": nbytes / med / 1e9, "hbm_fraction": nbytes / med / 1e9 / HBM_TBS}
        if ref is not None:
            t0 = time.perf_counter()
            with cf.ThreadPoolExecutor(os.cpu_count()) as ex:
                list(ex.map(lambda p: C_.run_ref(ref, p), pics))
            r["cpu_mc_ms"], r["cpu_threads"] = (time.perf_counter() - t0) * 1e3, os.cpu_count()
        # verification: one flush over the original pictures against the chained checker
        want = [C_.run_ref(mc_checker, p) for p in pics]
        M.apply_residual(checker, M.xvid_checker(), want, residual)
        for fr, pic in zip(g.frames, pics):
            for b, a in zip(fr, pic.frame):
                L.check(L.lib.avb200_memcpy_h2d(b.ptr, a.ctypes.data, a.nbytes, None), "h2d")
        arms["flush"][0]()
        device.sync()
        got = g.download()
        bad = [i for i in range(len(pics)) if M.first_diff(got[i], want[i])]
        r["verified"] = not bad and g.rejected() == 0
        if bad:
            r["mismatch"] = [M.first_diff(got[i], want[i]) for i in bad[:3]]
        results[kind] = r
        for a in arms:
            x = r[a]
            print("%s %-5s: %.3f ms median (best %.3f, spread %.1f %%), %.0f Mpixel/s, %.3f TB/s algorithmic = %.1f %% of %.2f TB/s"
                  % (kind, a, x["ms_median"], x["ms_best"], 100 * x["spread"], x["mpixel_s"], x["algo_TB_s"], 100 * x["hbm_fraction"], HBM_TBS))
        print("%s: %d records, %d residual batches / %d blocks; CPU reference MC %s; flush verified %s"
              % (kind, n_rec, len(residual), r["residual_blocks"],
                 "%.1f ms on %d threads" % (r["cpu_mc_ms"], r["cpu_threads"]) if "cpu_mc_ms" in r else "not available", r["verified"]))
    if args.out:
        with open(args.out, "w") as f:
            json.dump(results, f, indent=1)


if __name__ == "__main__":
    main()
