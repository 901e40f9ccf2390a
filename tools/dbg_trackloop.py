"""GPU box: the loop of tests/test_gpu_trackloop.py, repeated with freshly tuned detectors; on a divergence from the oracle the
sequence's detections go to trackloop_out/trackloop_fail_<k>.npz (replayable on CPU through the host simulator)."""
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PKG = os.path.join(ROOT, "yolov7-tracker_b200")
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(PKG, "tracker"))
sys.path.insert(1, PKG)
from oracle import trackers as OT  # noqa: E402
from basetrack import BaseTrack  # noqa: E402
from bytetrack import ByteTrack  # noqa: E402
from models.experimental import attempt_load  # noqa: E402
from utils.torch_utils import select_device  # noqa: E402
from utils.general import non_max_suppression, scale_coords  # noqa: E402


class Opts:
    conf_thresh = 0.2; track_buffer = 30; kalman_format = "default"; img_size = 256; iou_thresh = 0.5
    reid_model_path = ""; dhn_path = ""; gamma = 0.1; tracker = "bytetrack"; trace = False


def run(k):
    opts = Opts()
    device = select_device('0')
    model = attempt_load("seeded:0:256", map_location=device)
    rng = np.random.default_rng(2024)
    seqs = {}
    for name in ("seq_a", "seq_b"):
        base = rng.integers(0, 256, (256, 256, 3), dtype=np.uint8)
        seqs[name] = [np.ascontiguousarray(np.roll(base, (3 * j, 2 * j), axis=(0, 1))) for j in range(12)]
    BaseTrack._count = 0
    ids = OT.IdCounter()
    bad = 0
    for name, frames in seqs.items():
        tracker = ByteTrack(opts, frame_rate=30, gamma=opts.gamma)
        oracle = OT.TrackerOracle("bytetrack", ids=ids)
        hist = []
        id0 = ids.count
        for frame_id, img0_np in enumerate(frames, 1):
            img = torch.from_numpy(np.ascontiguousarray(img0_np[:, :, ::-1].transpose(2, 0, 1))).float().div_(255.0)[None]
            out = model(img.to(device))[0]
            out = non_max_suppression(out, 0.01, 0.45)[0]
            out[:, :4] = scale_coords(img.shape[2:], out[:, :4], img0_np.shape, ratio_pad=None).round()
            out = out[(out[:, 2] - out[:, 0] >= 1) & (out[:, 3] - out[:, 1] >= 1)]
            if JITTER:
                jit = ((torch.arange(out.shape[0] * 4, device=out.device, dtype=torch.float64).reshape(-1, 4) * 0.6180339887498949) % 1.0 - 0.5) * 0.4
                out[:, :4] += jit.to(out.dtype)
            cur = tracker.update(out, img0_np)
            dets_np = out.detach().cpu().numpy()
            hist.append(dets_np)
            exp = oracle.update(dets_np)
            cid = [t.track_id for t in cur]
            eid = [e[0] for e in exp]
            a = np.array([t.tlwh for t in cur]).reshape(-1, 4)
            b = np.array([e[1] for e in exp]).reshape(-1, 4)
            ok = cid == eid and (len(a) == 0 or np.allclose(a, b, rtol=1e-9, atol=1e-9, equal_nan=True))
            if not ok:
                bad += 1
                print("run %d %s frame %d DIVERGED: n %d/%d" % (k, name, frame_id, len(cid), len(eid)))
                if cid == eid:
                    rows = np.where(~np.isclose(a, b, rtol=1e-9, atol=1e-9, equal_nan=True).all(1))[0]
                    for r in rows:
                        print("   row %d id %d gpu %s oracle %s" % (r, cid[r], a[r], b[r]))
                else:
                    print("   ids gpu", cid[:40]); print("   ids orc", eid[:40])
                os.makedirs(os.path.join(ROOT, "trackloop_out"), exist_ok=True)
                np.savez(os.path.join(ROOT, "trackloop_out", "trackloop_fail_%d_%s.npz" % (k, name)), id0=id0, **{"f%d" % i: h for i, h in enumerate(hist)})
                break
    print("run %d: %s" % (k, "DIVERGED" if bad else "ok"))
    return bad


JITTER = "--jitter" in sys.argv

if __name__ == "__main__":
    n = int(sys.argv[1]) if len(sys.argv) > 1 and sys.argv[1].isdigit() else 4
    tot = sum(run(k) for k in range(n))
    print("diverged runs:", tot)
