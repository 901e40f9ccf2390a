"""StrongSORT's OSNet x0.25 extractor on the GPU: crops/s of b200track.osnet.OsnetExtractor against the same network in torch (oracle/osnet.py
on cuDNN, fp32 and fp16 channels-last) and the reference's recipe (per-crop host cv2.resize + Normalize + stack + H2D, then the torch
fp32 network), for n in {32, 256, 1024} crops of 128 x 256; network only (preprocessed input on the device) and frame + boxes -> features.
Also: kernel launches per forward, and a per-kernel time table (torch.profiler, a run of its own) with the FLOP and bytes each kernel kind
needs, computed from the shapes.  Seeded weights (oracle.osnet.seeded_state_dict).  Reads the card's name and power limit in the same run.

    python tools/osnet_bench.py --out DIR
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "yolov7-tracker_b200")):
    sys.path.insert(0, p)
from b200track.osnet import OsnetExtractor  # noqa: E402
from oracle import osnet as O  # noqa: E402

PEAK_BW, PEAK_F32 = 3.35e12, 67e12            # H100 SXM data sheet (700 W): HBM3 bytes/s, dense FP32 FLOP/s


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else torch.cuda.get_device_name()


def timed(fn, iters, warmup=3):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(iters):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / 1e3 / iters


def scene(seed, n, fh=720, fw=1280):
    rng = np.random.default_rng(seed)
    frame = np.ascontiguousarray(rng.integers(0, 256, (fh, fw, 3), dtype=np.uint8))
    x1, y1 = rng.uniform(0, fw - 40, n), rng.uniform(0, fh - 80, n)
    w, h = rng.uniform(20, 160, n), rng.uniform(40, 320, n)
    return frame, np.stack([x1, y1, np.minimum(x1 + w, fw), np.minimum(y1 + h, fh)], 1)


def reference_preprocess(frame, boxes):
    """strongsort.py:66-89's host path: slice, / 255, cv2.resize(dsize=(256, 128)), Normalize, stack, .cuda()"""
    import cv2
    mean, std = np.array([0.485, 0.456, 0.406], np.float32), np.array([0.229, 0.224, 0.225], np.float32)
    out = []
    for b in boxes:
        x1, y1, x2, y2 = [int(v) for v in b]
        r = cv2.resize(frame[y1:y2, x1:x2].astype(np.float32) / 255.0, dsize=(256, 128))
        out.append(torch.from_numpy(((r - mean) / std).transpose(2, 0, 1).copy()))
    return torch.stack(out).cuda()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True)
    ap.add_argument("--iters", type=int, default=20)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("osnet_bench needs a CUDA device")
    os.makedirs(args.out, exist_ok=True)
    torch.backends.cudnn.benchmark = True
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    sd = O.seeded_state_dict(0)
    sd32 = {k: v.cuda() for k, v in sd.items()}
    sd16 = {k: (v.half() if v.is_floating_point() else v) for k, v in sd32.items()}
    ext = OsnetExtractor(sd, device="cuda:0")
    res = {"card": card(), "launches_per_forward": ext.launches(), "rows": []}
    print(res["card"], "launches per forward:", res["launches_per_forward"], flush=True)
    for n in (32, 256, 1024):
        frame, boxes = scene(n, n)
        d_frame = torch.from_numpy(frame).cuda()
        x = reference_preprocess(frame, boxes)
        x16 = x.half().contiguous(memory_format=torch.channels_last)
        with torch.no_grad():
            row = {"n": n,
                   "ours_net_s": timed(lambda: ext.forward_nchw(x), args.iters),
                   "ours_frame_s": timed(lambda: ext.features_from_frame(d_frame, boxes), args.iters),
                   "torch_fp32_net_s": timed(lambda: O.forward(sd32, x), args.iters),
                   "torch_fp16_cl_net_s": timed(lambda: O.forward(sd16, x16), args.iters)}
            it = max(2, args.iters // 5)
            t0 = time.perf_counter()
            for _ in range(it):
                O.forward(sd32, reference_preprocess(frame, boxes))
            torch.cuda.synchronize()
            row["reference_recipe_frame_s"] = (time.perf_counter() - t0) / it
            ref = O.forward(sd32, x)
            f = ext.forward_nchw(x).double()
            row["min_cosine_vs_fp32"] = float(((f * ref.double()).sum(1) / (f.norm(dim=1) * ref.double().norm(dim=1))).min())
            row["max_rel_l2_vs_fp32"] = float(((f - ref.double()).norm(dim=1) / ref.double().norm(dim=1)).max())
        for k in list(row):
            if k.endswith("_s"):
                row[k.replace("_s", "_crops_per_s")] = n / row[k]
        res["rows"].append(row)
        print(json.dumps(row), flush=True)
    # per-kernel table at n = 256, profiler in a run of its own
    n = 256
    x = reference_preprocess(*scene(256, n))
    ext.forward_nchw(x)
    net = ext.last_net
    kinds = {}
    for name, flop, nbytes in net["kernels"]:
        k = kinds.setdefault(name, {"launches": 0, "flop": 0.0, "bytes": 0.0})
        k["launches"] += 1; k["flop"] += flop; k["bytes"] += nbytes
    from torch.profiler import ProfilerActivity, profile
    reps = 10
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(reps):
            ext.forward_nchw(x)
        torch.cuda.synchronize()
    times = {}
    for e in prof.key_averages():
        if "osnet_" in e.key or "image_nhwc16" in e.key:
            times[e.key] = (getattr(e, "device_time_total", None) or e.cuda_time_total) / 1e6 / reps
    table = []
    for name, k in kinds.items():
        t = sum(v for kk, v in times.items() if ("osnet_%s_kernel" % name.replace("pointwise_pool", "pointwise")) in kk)
        if name == "pointwise" or name == "pointwise_pool":
            pw = kinds.get("pointwise", {"flop": 0}), kinds.get("pointwise_pool", {"flop": 0})
            t *= k["flop"] / max(1.0, pw[0]["flop"] + pw[1]["flop"])       # one kernel serves both kinds: split its time by FLOP
        bound = max(k["flop"] / PEAK_F32, k["bytes"] / PEAK_BW)
        table.append({"kernel": name, "launches": k["launches"], "time_s": t, "gflop": k["flop"] / 1e9, "mbytes": k["bytes"] / 1e6,
                      "tflops": k["flop"] / t / 1e12 if t else None, "gbps": k["bytes"] / t / 1e9 if t else None,
                      "bound": "fp32" if k["flop"] / PEAK_F32 > k["bytes"] / PEAK_BW else "hbm", "share_of_peak": bound / t if t else None})
    res["kernels_n256"] = table
    res["profiler_kernels_n256_s"] = times
    for r in table:
        print(json.dumps(r), flush=True)
    with open(os.path.join(args.out, "osnet_bench.json"), "w") as f:
        json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
