"""GPU: op-level rooflines of the association branch -- BASELINE config C5 and SURVEY.md 8(d)'s "Kalman / IoU vs HBM peak".

    python tools/micro_bench.py [--dtype f32|f64] [--batch 64]

  * IoU cost + exact thresholded LAP for N = M in {64 ... 2048}, `batch` independent problems per launch (C5: boxes as in the
    synthetic streams, second set = first + N(0, 3) jitter, permuted; thresholds 0.9 and 0.5).  Algorithmic bytes: IoU reads
    16 (N + M) and writes e N M; LAP reads the matrix once (e N M).
  * Kalman predict / update / multi_gmc over 1 M tracks: 144 e / 148 e / 144 e bytes per track (e = 4 or 8).
Every kernel is timed with CUDA events after warm-up, L2 flushed between repetitions; GB/s against MEASURED_PEAKS.json.
"""
import argparse
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "yolov7-tracker_b200"))


def main():
    import torch
    from b200track import _lib as L
    from b200track.engine import Ops
    ap = argparse.ArgumentParser()
    ap.add_argument("--dtype", default="f32", choices=["f32", "f64"])
    ap.add_argument("--batch", type=int, default=64)
    ap.add_argument("--reps", type=int, default=10)
    args = ap.parse_args()
    dt, e = (L.F32, 4) if args.dtype == "f32" else (L.F64, 8)
    tdt = torch.float32 if e == 4 else torch.float64
    ops = Ops()
    dev = ops.device
    peaks = json.load(open(os.path.join(ROOT, "MEASURED_PEAKS.json"))) if os.path.exists(os.path.join(ROOT, "MEASURED_PEAKS.json")) else {}
    hbm = float(peaks.get("hbm_gbs", 6577.0))
    flush = torch.empty(256 << 20, dtype=torch.uint8, device=dev)

    def timed(fn, reps=args.reps):
        fn(); fn()
        torch.cuda.synchronize()
        tot = 0.0
        for _ in range(reps):
            flush.zero_()
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record(); fn(); b.record()
            torch.cuda.synchronize()
            tot += a.elapsed_time(b)
        return tot / reps

    rows = []
    rng = np.random.default_rng(5000)
    for n in (64, 128, 256, 512, 1024, 2048):
        B = args.batch
        c = rng.uniform(200, 1080, (B, n, 2)); wh = np.stack([rng.uniform(20, 80, (B, n)), rng.uniform(40, 160, (B, n))], -1)
        a = np.concatenate([c - wh / 2, c + wh / 2], -1)
        bb = a + rng.normal(0, 3, a.shape)
        for k in range(B):
            bb[k] = bb[k][rng.permutation(n)]
        ta, tb = ops.dev(a, tdt), ops.dev(bb, tdt)
        cost = torch.empty((B, n, n), dtype=tdt, device=dev)
        ms_iou = timed(lambda: ops.iou_cost(dt, ta, tb, out=cost))
        ws = ops.lap_workspace(dt, n, n, B)
        res = {}
        for thr in (0.9, 0.5):
            res[thr] = timed(lambda: ops.lap_solve(dt, cost, thr, workspace=ws), reps=max(3, args.reps // 2))
        iou_bytes = B * (32 * n + e * n * n)
        lap_bytes = B * e * n * n
        rows.append({"n": n, "batch": B, "iou_ms": ms_iou, "iou_gbps": iou_bytes / ms_iou / 1e6, "lap_ms_0.9": res[0.9], "lap_ms_0.5": res[0.5],
                     "lap_gbps_0.9": lap_bytes / res[0.9] / 1e6})
        print("N=M=%4d x%d: IoU %.3f ms = %7.1f GB/s (%.1f %% of %.0f) | LAP thr 0.9 %.3f ms = %7.1f GB/s, thr 0.5 %.3f ms"
              % (n, B, ms_iou, rows[-1]["iou_gbps"], 100 * rows[-1]["iou_gbps"] / hbm, hbm, res[0.9], rows[-1]["lap_gbps_0.9"], res[0.5]))
    T = 1 << 20
    meas = ops.dev(np.stack([rng.uniform(200, 1080, T), rng.uniform(200, 1080, T), rng.uniform(0.3, 0.8, T), rng.uniform(40, 160, T)], 1), tdt)
    mean, cov = ops.kalman_initiate(dt, L.FMT_BY_NAME["default"], meas)
    ms_p = timed(lambda: ops.kalman_predict(dt, L.FMT_BY_NAME["default"], mean, cov))
    mean, cov = ops.kalman_initiate(dt, L.FMT_BY_NAME["default"], meas)
    ms_u = timed(lambda: ops.kalman_update(dt, L.FMT_BY_NAME["default"], mean, cov, meas))
    mean, cov = ops.kalman_initiate(dt, L.FMT_BY_NAME["botsort"], meas)
    ms_g = timed(lambda: ops.gmc_apply(dt, mean, cov, [1.0, 0.0, 2.0, 0.0, 1.0, -1.5]))
    for name, ms, vals in (("kalman_predict", ms_p, 144), ("kalman_update", ms_u, 148), ("multi_gmc", ms_g, 144)):
        gbps = T * vals * e / ms / 1e6
        rows.append({"op": name, "tracks": T, "ms": ms, "gbps": gbps, "frac": gbps / hbm})
        print("%-15s %d tracks: %.3f ms = %7.1f GB/s = %.1f %% of %.0f GB/s" % (name, T, ms, gbps, 100 * gbps / hbm, hbm))
    print(json.dumps({"dtype": args.dtype, "hbm_peak_gbps": hbm, "rows": rows}))


if __name__ == "__main__":
    main()
