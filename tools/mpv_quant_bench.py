"""Throughput of the mpegvideo encoders' quantiser stage (ff_mpv_dct_quantize_batch_cuda) on one GPU, over sixteen 1080p 4:2:0 pictures
(783,360 8x8 blocks) in one call, timed with CUDA events after a warm-up, median and spread over repeats:
  plain    the fused inter path: diff_pixels + islow FDCT + ff_dct_quantize_c + clip + elimination.  Bytes per block: 64 read + 64 read
           (prediction) + 128 written (levels) + 4 written (last_index) + 8 (record) + 4 (offset) = 272; the share of the 3.35 TB/s HBM3
           data-sheet bandwidth is computed from that.
  trellis  the same with dct_quantize_trellis_c, against the reference's own dct_quantize_trellis_c (oracle/_ref/libmpvqref.so) run on the
           same blocks on every host core (one thread per core, each on its own share of the blocks).
Outputs are compared with the reference after the timed region.  Prints one JSON line (and writes it to --out when given).
usage: python tools/mpv_quant_bench.py [--reps 20] [--warmup 3] [--out result.json]"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import time
from concurrent.futures import ThreadPoolExecutor

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

HBM = 3.35e12


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--out")
    a = ap.parse_args()
    import libav_b200._lib as L
    from libav_b200 import device
    import mpv_quant_cases as M
    from test_gpu_mpv_quant import hd_pictures

    gpu_info = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                              capture_output=True, text=True).stdout.strip()
    L.init(0)
    lib = L.lib
    ref = M.ref_oracle()
    assert ref is not None, "the reference quantisers (oracle/_ref/libmpvqref.so) were not built"
    cur, rf, off, stride, chroma = hd_pictures(16, 5)
    n = len(off)
    rng = np.random.default_rng(6)
    recs = np.zeros(n, M.REC)
    mb = np.arange(n) // 6
    q = rng.integers(2, 12, n // 6 + 1)
    recs["qscale"], recs["chroma"], recs["dc_scale"] = q[mb], chroma, 8
    recs["lambda2"] = (q[mb].astype(np.int64) ** 2 * 109).astype(np.uint32)
    st = M.make_state(M.matrices_checker(), 0, M.FMT_H263, maxq=127, elim=(3, 4), seed=99)
    vlc = M.Vlc(9)
    h = lib.ff_mpv_quant_state_cuda(C.byref(st), C.byref(vlc.product()))
    assert h, L.last_error()
    d_cur, d_ref, d_off = device.DevBuf.from_numpy(cur), device.DevBuf.from_numpy(rf), device.DevBuf.from_numpy(off)
    d_rec = device.DevBuf.from_numpy(recs)
    d_blk, d_last = device.DevBuf(n * 128), device.DevBuf(n * 4)
    d_score = device.DevBuf.from_numpy(np.full(n, M.SCORE_UNSET, np.int32))     # where the trellis writes no coded_score it stays
    e0, e1 = lib.avb200_event_create(), lib.avb200_event_create()

    def launch(trellis):
        L.check(lib.ff_mpv_dct_quantize_batch_cuda(h, trellis, d_rec.ptr, d_cur.ptr, d_ref.ptr, d_off.ptr, None, stride, d_blk.ptr, n,
                                                   d_last.ptr, d_score.ptr, None, None), "quantize")

    def timed(trellis):
        for _ in range(a.warmup):
            launch(trellis)
        device.sync()
        ms = []
        for _ in range(a.reps):
            lib.avb200_event_record(e0, None)
            launch(trellis)
            lib.avb200_event_record(e1, None)
            lib.avb200_event_sync(e1)
            ms.append(lib.avb200_event_elapsed_ms(e0, e1))
        device.sync()
        return np.array(ms)

    blk = M.spatial(cur, rf, off, stride)
    out = {"gpu": gpu_info, "blocks": n, "reps": a.reps}
    for trellis in (0, 1):
        ms = timed(trellis)
        got = (d_blk.download(np.int16, (n, 64)), d_last.download(np.int32, (n,)), d_score.download(np.int32, (n,)))
        med = float(np.median(ms))
        key = "trellis" if trellis else "plain"
        out[key] = {"ms_median": round(med, 4), "ms_min": round(float(ms.min()), 4), "ms_max": round(float(ms.max()), 4),
                    "spread_pct": round(100 * float(ms.max() - ms.min()) / med, 2), "blocks_per_s": n / (med * 1e-3)}
        if not trellis:
            out[key]["bytes_per_block"] = 272
            out[key]["hbm_share_pct"] = round(100 * n * 272 / (med * 1e-3) / HBM, 2)
        # the reference on every host core, on the same blocks (timed), then compared
        cores = os.cpu_count()
        chunks = np.array_split(np.arange(n), cores)
        res = [None] * cores

        def work(k):
            idx = chunks[k]
            res[k] = ref.run(st, vlc, trellis, recs[idx], blk[idx])

        t0 = time.perf_counter()
        with ThreadPoolExecutor(cores) as ex:
            list(ex.map(work, range(cores)))
        cpu_s = time.perf_counter() - t0
        want = tuple(np.concatenate([r[i] for r in res]) for i in range(4))
        skip = M.undefined_blocks(st, vlc, trellis, recs, blk)
        M.compare(key, want, *got, trellis, skip=skip)
        out[key].update({"reference_cores": cores, "reference_blocks_per_s": n / cpu_s, "speedup_vs_reference": round(n / (med * 1e-3) / (n / cpu_s), 1),
                         "bitexact": True, "undefined_blocks_skipped": int(skip.sum())})
    lib.ff_mpv_quant_state_free_cuda(h)
    line = json.dumps(out)
    print(line)
    if a.out:
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
