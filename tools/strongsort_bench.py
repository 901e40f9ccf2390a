"""StrongSORT on the device: the fused step against BoT-SORT with ReID on the same stream, and the feature-distance kernel.

    python tools/strongsort_bench.py [--seq 8] [--objects 300] [--frames 120]

Prints the card's name and power limit, then
  * the step time (CUDA events around TrackEngine.step_device, after warm-up) for S sequences of a C4-sized stream (300 objects,
    512-d features): StrongSORT (feature distances + step) and BoT-SORT with ReID (feat_dim 512) on the same detections and features;
  * the distance kernel alone (b2t_feature_distance) at rows = cols = 300, D = 512, S sequences: time, fp64 instructions per second
    (3 per element and dimension: subtract, multiply, add) against the data sheet's 34 TFLOP/s fp64 for the H100 SXM, i.e. about
    17 T DP instructions/s since that figure counts an FMA as two flops.
Nothing is written."""
import argparse
import ctypes as C
import os
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "yolov7-tracker_b200"))
from b200track import _lib as L                       # noqa: E402
from b200track.engine import TrackEngine              # noqa: E402
from b200track.synth import make_strongsort_stream    # noqa: E402

DP_INSTR_PER_S = 34e12 / 2        # H100 SXM data sheet, fp64 non-tensor 34 TFLOP/s with FMA = 2 flops


def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                              text=True).stdout.strip().splitlines()[0]
    except Exception:
        return torch.cuda.get_device_name()


def pack(frames, feats, S, dmax, D):
    n = len(frames[0])
    dets = torch.zeros((n, S, dmax, 6), dtype=torch.float32)
    fe = torch.zeros((n, S, dmax, D), dtype=torch.float32)
    cnt = torch.zeros((n, S), dtype=torch.int32)
    for s in range(S):
        for i in range(n):
            k = len(frames[s][i])
            dets[i, s, :k] = torch.from_numpy(frames[s][i]); fe[i, s, :k] = torch.from_numpy(feats[s][i]); cnt[i, s] = k
    return dets.cuda(), fe.cuda(), cnt.cuda()


def time_steps(eng, dets, fe, cnt, warps, warm):
    out = torch.zeros((eng.S, eng.cap, L.OUT_COLS), dtype=torch.float64, device="cuda")
    stat = torch.zeros((eng.S, L.STAT_WORDS), dtype=torch.int32, device="cuda")
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
    n = dets.shape[0]
    for i in range(n):
        if i == warm:
            ev[0].record()
        eng.step_device(dets[i], cnt[i], out, stat, warps=warps[i], feats=fe[i])
    ev[1].record()
    torch.cuda.synchronize()
    assert int(stat[:, L.STAT_ERR].max()) == 0
    return ev[0].elapsed_time(ev[1]) * 1e3 / (n - warm)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--seq", type=int, default=8)
    ap.add_argument("--objects", type=int, default=300)
    ap.add_argument("--frames", type=int, default=120)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("strongsort_bench needs a CUDA device: not measured")
    S, D, dmax = a.seq, 512, 512
    print("card: %s" % card())
    streams = [make_strongsort_stream(1000 + s, a.frames, a.objects, D) for s in range(S)]
    dets, fe, cnt = pack([st[0] for st in streams], [st[1] for st in streams], S, dmax, D)
    warps = torch.from_numpy(np.stack([st[2] for st in streams], 1).reshape(a.frames, S, 6).astype(np.float32).astype(np.float64)).cuda()
    warm = min(20, a.frames // 4)
    res = {}
    for kind in ("strongsort", "botsort"):
        eng = TrackEngine(kind, n_seq=S, cap=1024, dmax=dmax, feat_dim=D)
        res[kind] = time_steps(eng, dets, fe, cnt, warps, warm)
    print("step, %d sequences, %d objects, %d-d features: StrongSORT %.1f us, BoT-SORT with ReID %.1f us (mean over %d frames)"
          % (S, a.objects, D, res["strongsort"], res["botsort"], a.frames - warm))
    lib = L.load()
    n = m = 300
    x = torch.randn((S, n, D), device="cuda") / 22.6
    y = torch.randn((S, m, D), device="cuda") / 22.6
    o = torch.empty((S, n, m), dtype=torch.float64, device="cuda")
    st = C.c_void_p(torch.cuda.current_stream().cuda_stream)
    call = lambda: L.check(lib, lib.b2t_feature_distance(x.data_ptr(), n, y.data_ptr(), m, D, o.data_ptr(), S, st))   # noqa: E731
    for _ in range(10):
        call()
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
    reps = 200
    ev[0].record()
    for _ in range(reps):
        call()
    ev[1].record()
    torch.cuda.synchronize()
    us = ev[0].elapsed_time(ev[1]) * 1e3 / reps
    instr = 3.0 * S * n * m * D
    print("distance kernel, %d x %d x %d x %d sequences: %.1f us, %.2f T DP instructions/s = %.1f %% of the data sheet's %.0f T/s"
          % (n, m, D, S, us, instr / us * 1e-6, 100 * instr / us * 1e6 / DP_INSTR_PER_S, DP_INSTR_PER_S * 1e-12))


if __name__ == "__main__":
    main()
