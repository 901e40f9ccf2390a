"""GPU box: cost of BoT-SORT with ReID inside TrackingPipeline, one JSON line.

The C4 end-to-end configuration of bench_pipeline.py -- twin YOLOv7-w6 at 1280 x 1280, batch 8, the headline's uint8 noise frames
resident in HBM, BoT-SORT with the camera-motion warp estimated on the GPU -- in four variants, alternated in this process (three timed
runs each, every shape warmed up first):
  no_reid        the pipeline without appearance
  batch_full     ReID, batch-statistics BatchNorm per sequence, reid_cap = S * dmax (cannot overflow)
  batch_tight    the same at the next multiple of 256 above the largest crop count seen in warm-up
  running        ReID with running-statistics BatchNorm (folded into the convs), reid_cap = S * dmax
Each run: device events around `steps` pipeline steps ending in flush() (a synchronise).  Also: the ReID chain alone (crop list + crop
cut + extractor graph) timed with CUDA events, valid crops per step and the padding fraction, the extractor's device memory, and the
card's name, power limit and SM clock.

The seeded random-init detector emits boxes that round to zero width or height, some at score 1.0 (the reference's own note at
botsort.py:283, "why some bboxs has 0 area"): no conf_thresh avoids them, and the pipeline refuses such a det_high crop as the reference
exits on it.  So before timing the stream is scanned and the count at conf_thresh 0.2 is reported ("det_high_refused_at_0.2"), and in
every variant every NMS row is widened to at least 2 px inside the frame on the tracker stream before the crop list, GMC and the step
("boxes_widened": true).  The count is per pool of frames the bench cycles through.

    python tools/reid_pipeline_bench.py [--steps 30] [--reps 3] [--out FILE]
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PKG = os.path.join(ROOT, "yolov7-tracker_b200")
sys.path.insert(0, ROOT)
sys.path.insert(0, PKG)
import torch  # noqa: E402
from b200track import _lib as L  # noqa: E402


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                           text=True, timeout=30).stdout.strip().splitlines()[0]
        name, power, sm, sm_max = [v.strip() for v in q.split(",")]
    except Exception:
        name, power, sm, sm_max = torch.cuda.get_device_name(0), "unknown", "unknown", "unknown"
    return {"name": name, "power_limit": power, "sm_clock_now": sm, "sm_clock_max": sm_max}


def refused_rows(d, c, thr, h, w):
    """det_high rows (score >= float32(thr)) whose crop the reference could not cut: empty after int() + slicing, or a negative
    coordinate; returns (count, best score of any such row whatever its score)"""
    n, best = 0, -np.inf
    for s in range(len(c)):
        r = d[s, :c[s]]
        t = np.trunc(r[:, :4].astype(np.float64))
        bad = (t < 0).any(1) | (np.minimum(t[:, 2], w) - np.minimum(t[:, 0], w) < 1) | (np.minimum(t[:, 3], h) - np.minimum(t[:, 1], h) < 1)
        n += int((bad & (r[:, 4] >= np.float32(thr))).sum())
        if bad.any():
            best = max(best, float(r[bad, 4].max()))
    return n, best


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=30)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--batch", type=int, default=8)
    ap.add_argument("--img", type=int, default=1280)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "needs a CUDA device: there is no CPU fallback"
    import bench_pipeline as BP
    from b200track.detector import DetectorW6
    from b200track.engine import TrackEngine
    from b200track.gmc import GmcEstimator
    from b200track.pipeline import TrackingPipeline
    from b200track.reid import ReidExtractor
    from b200track.w6 import calibrated_state_dict
    from oracle import reid as R
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    B, img = args.batch, args.img
    sd = calibrated_state_dict(0, img, dev)
    dets = [DetectorW6(sd, batch=B, img_size=img, device=dev, use_graph=True) for _ in range(2)]
    for d in dets:
        d.set_source_frames((img, img))
    frames = [torch.from_numpy(f).to(dev) for f in BP.make_frames(B, img, 1000)]
    dmax = dets[0].max_det
    # ---- the stream's refused det_high crops at the default threshold
    d0 = dets[0]
    refused, best = 0, -np.inf
    for f in frames:
        d0.src_u8.copy_(f)
        d0.ingest_u8_launch()
        for fn, _, _ in d0.ops[1:]:
            fn()
        d0._nms_launch(True)
        torch.cuda.synchronize()
        n, b = refused_rows(d0.out.cpu().numpy(), d0.out_count.cpu().numpy(), 0.2, img, img)
        refused += n
        best = max(best, b)
    conf = 0.2
    rsd = R.seeded_state_dict(6)
    ext = {"batch": ReidExtractor(rsd, device=dev, bn_mode="batch"), "running": ReidExtractor(rsd, device=dev, bn_mode="running")}

    def widen(d):
        x1 = d[..., 0].clamp(max=img - 2); y1 = d[..., 1].clamp(max=img - 2)
        d[..., 0] = x1; d[..., 1] = y1
        d[..., 2] = d[..., 2].maximum(x1 + 2); d[..., 3] = d[..., 3].maximum(y1 + 2)

    def make(mode, cap):
        eng = TrackEngine("botsort", n_seq=B, dtype="f64", cap=1152, dmax=dmax, device=dev, conf_thresh=conf, feat_dim=512 if mode else 0)
        gmc = GmcEstimator(B, img, img, 2, max_kp=32768, device=dev)
        pipe = TrackingPipeline(dets, eng, out_rows=1152, gmc=gmc, reid=ext[mode] if mode else None, reid_cap=cap if mode else None)
        # the NMS rows widened on the tracker stream before anything reads them: GMC and the step (no ReID), the crop list (ReID)
        est = gmc.estimate_prepared
        gmc.estimate_prepared = lambda k, d, c, **kw: (widen(d), est(k, d, c, **kw))[1]
        if mode:
            cut = pipe.reid_net.cut
            pipe.reid_net.cut = lambda fr, d, c, t: (widen(d), cut(fr, d, c, t))[1]
        return pipe

    def warm(pipe, n=8):
        totals = []
        for k in range(n):
            r = pipe.step(frames[k % len(frames)])
            if r is not None and pipe.reid_net is not None:
                totals.append(int(pipe.h_rstat[pipe.n & 1][B]))
        pipe.flush()
        if pipe.reid_net is not None:
            totals.append(int(pipe.h_rstat[(pipe.n - 1) & 1][B]))
        torch.cuda.synchronize()
        return totals

    def timed(pipe):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize()
        e0.record(pipe.s_copy)
        for k in range(args.steps):
            pipe.step(frames[k % len(frames)])
        pipe.flush()
        e1.record(pipe.s_trk)
        torch.cuda.synchronize()
        return e0.elapsed_time(e1) / args.steps

    pipes, seen = {}, {}
    pipes["no_reid"] = make(None, None); warm(pipes["no_reid"])
    pipes["batch_full"] = make("batch", B * dmax); seen["batch_full"] = warm(pipes["batch_full"])
    tight = (max(seen["batch_full"]) // 256 + 1) * 256
    pipes["batch_tight"] = make("batch", tight); seen["batch_tight"] = warm(pipes["batch_tight"])
    pipes["running"] = make("running", B * dmax); seen["running"] = warm(pipes["running"])
    runs = {k: [] for k in pipes}
    for _ in range(args.reps):
        for k, p in pipes.items():
            runs[k].append(timed(p))
    # ---- the ReID chain alone on the last frame's NMS output: crop list + crop cut + extractor graph, CUDA events over 10 calls
    chain = {}
    s = torch.cuda.Stream(device=dev)
    for k in ("batch_full", "batch_tight", "running"):
        rn = pipes[k].reid_net
        with torch.cuda.stream(s):
            for _ in range(2):
                rn.cut(dets[1].src_u8, dets[1].out, dets[1].out_count, conf); rn.run()
            torch.cuda.synchronize()
            rn.raise_for_status(rn.status.cpu().numpy())
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record(s)
            for _ in range(10):
                rn.cut(dets[1].src_u8, dets[1].out, dets[1].out_count, conf); rn.run()
            b.record(s)
        torch.cuda.synchronize()
        chain[k] = {"ms": a.elapsed_time(b) / 10, "cap": rn.cap, "extractor_bytes": rn.bytes}
    res = {"tool": "reid_pipeline_bench", "card": card(), "config": "C4 end to end: twin YOLOv7-w6 %dx%d, batch %d, noise frames, BoT-SORT + GPU GMC" % (img, img, B),
           "steps_per_run": args.steps, "det_high_refused_at_0.2": refused, "best_score_of_a_refused_box": best, "conf_thresh": conf,
           "boxes_widened": True, "variants": {}}
    for k in pipes:
        ms = runs[k]
        v = {"ms_per_step": ms, "frames_per_s": [B * 1e3 / m for m in ms]}
        if k in seen:
            t = np.array(seen[k], np.float64)
            cap = pipes[k].reid_net.cap
            v.update({"reid_cap": cap, "valid_crops_per_step_mean": float(t.mean()), "valid_crops_per_step_max": int(t.max()),
                      "padding_fraction": float(1.0 - t.mean() / cap), "reid_chain_alone_ms": chain[k]["ms"],
                      "extractor_bytes": chain[k]["extractor_bytes"]})
        res["variants"][k] = v
    line = json.dumps(res)
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
