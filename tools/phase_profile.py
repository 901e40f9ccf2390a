"""GPU: per-phase SM-cycle breakdown of track_step_kernel (stat[16..32)) and throughput vs #sequences."""
import os, sys, json
import numpy as np
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, "yolov7-tracker_b200"))
import torch
from b200track import _lib as L
from b200track.engine import TrackEngine
from b200track.synth import make_stream, pack_frames

NAMES = ["P0 dets", "P1 lists", "P2 predict", "P3 boxes", "P4 csr1", "P5 lap1", "P6 apply1", "P7 assoc2", "P8 assoc3",
         "P9 births", "P10 lists", "P11 dedup", "P12 output"]

def run(kind, S, dtype, frames=60, warm=60, nobj=300, dmax=512, cap=1024):
    base = [pack_frames(make_stream(3000 + s, warm + frames, nobj)[0], dmax) for s in range(min(S, 8))]
    dets = np.stack([base[s % len(base)][0] for s in range(S)], 1); cnt = np.stack([base[s % len(base)][1] for s in range(S)], 1)
    dev = torch.device("cuda:0")
    eng = TrackEngine(kind, n_seq=S, dtype=dtype, cap=cap, dmax=dmax)
    d_dets = torch.from_numpy(dets).to(dev); d_cnt = torch.from_numpy(cnt).to(dev)
    d_out = torch.zeros((S, 512, L.OUT_COLS), dtype=torch.float64, device=dev)
    d_stat = torch.zeros((warm + frames, S, L.STAT_WORDS), dtype=torch.int32, device=dev)
    for f in range(warm):
        eng.step_device(d_dets[f], d_cnt[f], d_out, d_stat[f])
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for f in range(warm, warm + frames):
        eng.step_device(d_dets[f], d_cnt[f], d_out, d_stat[f])
    e1.record(); torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / frames
    st = d_stat[warm:].cpu().numpy()
    assert st[:, :, L.STAT_ERR].max() == 0
    ph = st[:, :, L.STAT_PHASE0:L.STAT_PHASE0 + 13].astype(np.float64).mean(axis=(0, 1))
    return ms, ph, st

if __name__ == "__main__":
    kind = sys.argv[1] if len(sys.argv) > 1 else "bytetrack"
    for dtype in ("f64", "f32"):
        ms, ph, st = run(kind, 4, dtype)
        print("== %s %s S=4: %.1f us/step (warm L2, back-to-back) -> %.0f frames/s" % (kind, dtype, ms * 1e3, 4 / ms * 1e3))
        tot = ph.sum()
        for n, c in zip(NAMES, ph):
            print("   %-12s %9.0f cyc  %5.1f%%" % (n, c, 100 * c / tot))
        print("   total %.0f cyc; pool %.0f hi %.0f | assoc1: edges %.0f, rows left after kernelisation %.1f, deferred once %.1f, twice %.1f"
              % (tot, st[:, :, L.STAT_NPOOL].mean(), st[:, :, L.STAT_NHI].mean(), st[:, :, 15].mean(), st[:, :, 12].mean(), st[:, :, 13].mean(), st[:, :, 14].mean()))
        sub = st[:, :, L.STAT_SUB0:L.STAT_SUB0 + 16].astype(np.float64).mean(axis=(0, 1))
        print("   csr1 sub: colstats %.0f | sort %.0f | count %.0f | scan %.0f | list %.0f | iou %.0f" % tuple(sub[:6]))
        print("   lap1 sub: init %.0f | kernelize %.0f | compact %.0f | labels %.0f | solve %.0f" % tuple(sub[8:13]))
    for S in (1, 4, 132):
        ms, ph, st = run(kind, S, "f64", frames=30)
        print("S=%4d  %.1f us/step  %.0f frames/s" % (S, ms * 1e3, S / ms * 1e3))
