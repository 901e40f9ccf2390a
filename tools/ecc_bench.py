"""GPU box: ECC camera-motion estimation (b200track.gmc.EccEstimator, csrc/b2t_ecc.cu) against the reference's host OpenCV calls.

Prints one JSON line: the device name and its power limit (read in this run), ms per ``estimate`` call by CUDA events after warm-up
for n_seq in {1, 8} at 1280 x 720 and 1920 x 1080 with the iterations each call ran, and the host arm -- the four OpenCV calls
GMC.applyEcc makes (cvtColor, GaussianBlur, resize, findTransformECC; tracker/botsort.py:82-105) on one frame, with OpenCV's thread
count.  Every timed call aligns the same moved frame to the same template, so each repeats the same iterations.
``python tools/ecc_bench.py [reps]``"""
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "yolov7-tracker_b200")):
    sys.path.insert(0, p)
import numpy as np  # noqa: E402
import torch  # noqa: E402
from b200track.gmc import EccEstimator  # noqa: E402
from b200track.synth import textured_frame  # noqa: E402


def power_limit_w():
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader,nounits", "-i", "0"], capture_output=True, text=True, timeout=20)
        return float(r.stdout.strip().splitlines()[0])
    except Exception:
        return None


def frames_for(h, w, n_seq):
    base = [textured_frame(500 + s, h, w, n_rect=900) for s in range(n_seq)]
    moved = [np.ascontiguousarray(np.roll(b, (3, -5), (0, 1))) for b in base]
    return np.stack(base), np.stack(moved)


def gpu_arm(h, w, n_seq, reps):
    a, b = frames_for(h, w, n_seq)
    est = EccEstimator(n_seq, h, w)
    fa, fb = torch.from_numpy(a).cuda(), torch.from_numpy(b).cuda()
    est.estimate(fa)
    for _ in range(3):
        est.estimate(fb)
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        est.estimate(fb)
    e1.record()
    torch.cuda.synchronize()
    st = est.stat.cpu().numpy()
    return {"h": h, "w": w, "n_seq": n_seq, "ms_per_call": e0.elapsed_time(e1) / reps, "iterations": [int(v) for v in st[:, 0]],
            "flags": [int(v) for v in st[:, 5]]}


def host_arm(h, w, reps):
    try:
        import cv2
    except ImportError:
        return {"h": h, "w": w, "ms_per_frame": None, "note": "OpenCV not installed"}
    a, b = frames_for(h, w, 1)

    def prep(f):
        g = cv2.cvtColor(f, cv2.COLOR_BGR2GRAY)
        g = cv2.GaussianBlur(g, (3, 3), 1.5)
        return cv2.resize(g, (w // 2, h // 2))
    tmpl = prep(a[0])
    crit = (cv2.TERM_CRITERIA_EPS | cv2.TERM_CRITERIA_COUNT, 100, 1e-5)
    times = []
    for _ in range(reps + 1):
        t0 = time.perf_counter()
        H = np.eye(2, 3, dtype=np.float32)
        cv2.findTransformECC(tmpl, prep(b[0]), H, cv2.MOTION_EUCLIDEAN, crit, None, 1)
        times.append(time.perf_counter() - t0)
    return {"h": h, "w": w, "ms_per_frame": 1e3 * float(np.median(times[1:])), "threads": cv2.getNumThreads(), "opencv": cv2.__version__}


def main():
    reps = int(sys.argv[1]) if len(sys.argv) > 1 else 20
    out = {"bench": "ecc_estimate", "device": torch.cuda.get_device_name(0), "power_limit_w": power_limit_w(), "gpu": [], "host": []}
    for h, w in ((720, 1280), (1080, 1920)):
        for n_seq in (1, 8):
            out["gpu"].append(gpu_arm(h, w, n_seq, reps))
        out["host"].append(host_arm(h, w, max(3, reps // 5)))
    print(json.dumps(out))


if __name__ == "__main__":
    main()
