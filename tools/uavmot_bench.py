"""UAVMOT on the device: the fused step against ByteTrack's on the same stream, and the structure entries alone.

    python tools/uavmot_bench.py [--seq 4] [--objects 300] [--frames 160]

Prints the card's name and power limit, then one JSON line with
  * the step time (CUDA events around TrackEngine.step_device, after warm-up) for S sequences of the C3 stream (300 objects): the
    UAVMOT kind and the ByteTrack kind on the same detections, alternated;
  * b2t_structure_vectors on a 300-point track set and b2t_structure_distance at 300 x 300, each alone.
  * the CPU time per frame of the project's own restatement of UAVMOT.update (tests/uavmot_oracle.py, one core, the first sequence,
    --cpu-frames frames after the warm-up), labelled "port" as bench.py labels numbers that do not come from the reference's code:
    the reference's tracker/uavmot.py is not packed for the GPU machines.
Nothing is written."""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "yolov7-tracker_b200"))
from b200track import _lib as L                       # noqa: E402
from b200track.engine import TrackEngine, ops         # noqa: E402
from b200track.synth import make_stream               # noqa: E402


def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                              text=True).stdout.strip().splitlines()[0]
    except Exception:
        return torch.cuda.get_device_name()


def time_steps(kind, dets, cnt, S, warm):
    eng = TrackEngine(kind, n_seq=S, cap=1024, dmax=dets.shape[2])
    out = torch.zeros((S, eng.cap, L.OUT_COLS), dtype=torch.float64, device="cuda")
    stat = torch.zeros((S, L.STAT_WORDS), dtype=torch.int32, device="cuda")
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
    for i in range(dets.shape[0]):
        if i == warm:
            ev[0].record()
        eng.step_device(dets[i], cnt[i], out, stat)
    ev[1].record()
    torch.cuda.synchronize()
    assert int(stat[:, L.STAT_ERR].max()) == 0
    return ev[0].elapsed_time(ev[1]) * 1e3 / (dets.shape[0] - warm)


def time_call(fn, reps=200):
    fn()
    torch.cuda.synchronize()
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
    ev[0].record()
    for _ in range(reps):
        fn()
    ev[1].record()
    torch.cuda.synchronize()
    return ev[0].elapsed_time(ev[1]) * 1e3 / reps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--seq", type=int, default=4)
    ap.add_argument("--objects", type=int, default=300)
    ap.add_argument("--frames", type=int, default=160)
    ap.add_argument("--warmup", type=int, default=60)
    ap.add_argument("--cpu-frames", type=int, default=10)
    a = ap.parse_args()
    streams = [make_stream(1000 + s, a.frames, n_obj=a.objects)[0] for s in range(a.seq)]
    dmax = max(len(f) for st in streams for f in st)
    dets = torch.zeros((a.frames, a.seq, dmax, 6), dtype=torch.float32)
    cnt = torch.zeros((a.frames, a.seq), dtype=torch.int32)
    for s, st in enumerate(streams):
        for i, f in enumerate(st):
            dets[i, s, :len(f)] = torch.from_numpy(f)
            cnt[i, s] = len(f)
    dets, cnt = dets.cuda(), cnt.cuda()
    res = {"card": card(), "seq": a.seq, "objects": a.objects, "timed_frames": a.frames - a.warmup}
    for kind in ("uavmot", "bytetrack", "uavmot", "bytetrack"):           # alternated
        res.setdefault("step_us_" + kind, []).append(round(time_steps(kind, dets, cnt, a.seq, a.warmup), 1))
    o = ops()
    rng = np.random.default_rng(0)
    pts = o.dev(rng.uniform(200, 1080, (a.objects, 2)), torch.float64)
    sv = o.structure_vectors(pts)
    res["structure_vectors_us"] = round(time_call(lambda: o.structure_vectors(pts)), 1)
    res["structure_distance_us"] = round(time_call(lambda: o.structure_distance(sv, sv)), 1)
    sys.path.insert(0, ROOT)
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    import time
    from uavmot_oracle import UavmotOracle
    orc = UavmotOracle()
    for f in streams[0][:a.warmup]:
        orc.update(f)
    t0 = time.perf_counter()
    for f in streams[0][a.warmup:a.warmup + a.cpu_frames]:
        orc.update(f)
    res["cpu_baseline"] = {"kind": "port", "ms_per_frame": round((time.perf_counter() - t0) * 1e3 / a.cpu_frames, 1), "cores": 1,
                           "what": "tests/uavmot_oracle.py UavmotOracle.update (the CPU restatement the step is checked against), one sequence"}
    print(json.dumps(res))


if __name__ == "__main__":
    main()
