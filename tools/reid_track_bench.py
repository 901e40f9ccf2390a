"""GPU box: cost of BoT-SORT's appearance path, one JSON line.

  fused step   the C4 tracking load -- 8 sequences, about 420 detections per frame, features already on the device -- through one
               TrackEngine without features (b2t_tracker_step) and one with 512-d features (b2t_tracker_step_feat), alternated
               stream by stream in this process and timed with CUDA events around every step;
  drop-in      BoTSORT(use_apperance_model=True) with a seeded ReidExtractor on a 1280 x 1280 uint8 frame with about 250
               high-score detections: extractor + fused step per update, host clock around synchronised updates.
The card's name and power limit are printed and stored in the line: a time means something only next to them.

    python tools/reid_track_bench.py [--frames 40] [--reps 3] [--out FILE]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PKG = os.path.join(ROOT, "yolov7-tracker_b200")
sys.path.insert(0, ROOT)
sys.path.insert(0, PKG)
import torch  # noqa: E402
from b200track import _lib as L  # noqa: E402
from b200track.engine import TrackEngine  # noqa: E402
from b200track.synth import make_reid_stream  # noqa: E402


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True,
                           timeout=30).stdout.strip().splitlines()[0]
        name, power = [v.strip() for v in q.split(",")]
    except Exception:
        name, power = torch.cuda.get_device_name(0), "unknown"
    return name, power


def fused_step(frames_n, reps, dim=512, S=8, n_obj=490):
    dev = torch.device("cuda:0")
    streams = [make_reid_stream(400 + s, frames_n, n_obj, dim) for s in range(S)]
    dmax = 576
    dets = torch.zeros((frames_n, S, dmax, 6), dtype=torch.float32)
    feats = torch.zeros((frames_n, S, dmax, dim), dtype=torch.float32)
    cnt = torch.zeros((frames_n, S), dtype=torch.int32)
    warps = torch.zeros((frames_n, S, 6), dtype=torch.float64)
    for s, (fr, fe, wa) in enumerate(streams):
        for i in range(frames_n):
            n = len(fr[i])
            dets[i, s, :n] = torch.from_numpy(fr[i]); feats[i, s, :n] = torch.from_numpy(fe[i]); cnt[i, s] = n
            warps[i, s] = torch.from_numpy(wa[i].reshape(6))
    dets, feats, cnt, warps = dets.to(dev), feats.to(dev), cnt.to(dev), warps.to(dev)
    engines = {0: TrackEngine("botsort", n_seq=S, cap=1152, dmax=dmax), dim: TrackEngine("botsort", n_seq=S, cap=1152, dmax=dmax, feat_dim=dim)}
    out = {k: torch.zeros((S, 1152, L.OUT_COLS), dtype=torch.float64, device=dev) for k in engines}
    stat = {k: torch.zeros((S, L.STAT_WORDS), dtype=torch.int32, device=dev) for k in engines}
    times = {k: [] for k in engines}
    napp = 0
    ev = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(frames_n)]
    for rep in range(reps + 1):                                      # rep 0 warms both up
        for k, eng in engines.items():
            eng.reset()
            for i in range(frames_n):
                ev[i][0].record()
                eng.step_device(dets[i], cnt[i], out[k], stat[k], warps=warps[i], feats=feats[i] if k else None)
                ev[i][1].record()
            torch.cuda.synchronize()
            if int(stat[k][:, L.STAT_ERR].max()):
                raise RuntimeError("capacity exceeded in the C4 stream (feat_dim %d)" % k)
            if rep and k:
                napp += int(stat[k][:, L.STAT_NAPP].sum())
            if rep:
                times[k].append(float(np.sum([a.elapsed_time(b) for a, b in ev[2:]])) / (frames_n - 2))
    per_frame = float(np.mean([len(f) for st in streams for f in st[0]]))
    return {"dets_per_seq_frame": round(per_frame, 1), "feat_dim": dim,
            "step_ms_feat0": [round(t, 4) for t in times[0]], "step_ms_feat": [round(t, 4) for t in times[dim]],
            "step_ms_feat0_median": round(float(np.median(times[0])), 4), "step_ms_feat_median": round(float(np.median(times[dim])), 4),
            "appearance_pairs_last_frame": napp // reps}


def dropin(frames_n, n_obj=300):
    from oracle import reid as R
    from b200track.reid import ReidExtractor
    sys.path.insert(0, os.path.join(PKG, "tracker"))
    from basetrack import BaseTrack
    from botsort import BoTSORT

    class Opts:
        conf_thresh = 0.2; track_buffer = 30; kalman_format = "botsort"; img_size = 1280; iou_thresh = 0.5
        reid_model_path = ""; dhn_path = ""

    frames, _, _ = make_reid_stream(77, frames_n, n_obj, 512)
    img = np.random.default_rng(1).integers(0, 256, (1280, 1280, 3), dtype=np.uint8)
    BaseTrack._count = 0
    trk = BoTSORT(Opts(), use_GMC=False)
    trk.use_apperance_model = True
    trk.reid_model = ReidExtractor(R.seeded_state_dict(6), bn_mode="batch")
    ts = []
    for i, f in enumerate(frames):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        trk.update(f.copy(), img)
        torch.cuda.synchronize()
        if i >= 3:
            ts.append((time.perf_counter() - t0) * 1e3)
    nhi = float(np.mean([(f[:, 4] >= np.float32(0.2)).sum() for f in frames]))
    return dict(dropin_high_dets=round(nhi, 1), dropin_frame_ms_median=round(float(np.median(ts)), 3),
                dropin_frame_ms_p90=round(float(np.percentile(ts, 90)), 3))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=40)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--out", default="")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("reid_track_bench needs a CUDA device")
    name, power = card()
    print("card: %s, power limit %s" % (name, power))
    res = dict(card=name, power_limit=power)
    res.update(fused_step(a.frames, a.reps))
    res.update(dropin(a.frames))
    line = json.dumps(res)
    print(line)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "a") as fh:
            fh.write(line + "\n")


if __name__ == "__main__":
    main()
