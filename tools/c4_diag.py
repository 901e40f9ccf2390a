import os, sys, numpy as np, torch
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, "yolov7-tracker_b200"))
from b200track import _lib as L
from b200track.detector import DetectorW6
from b200track.engine import TrackEngine
from b200track.gmc import GmcEstimator
from b200track.synth import textured_frame
from b200track.w6 import calibrated_state_dict
B, S = 8, 1280
dev = torch.device("cuda:0")
sd = calibrated_state_dict(0, S, dev)
det = DetectorW6(sd, batch=B, img_size=S, device=dev, use_graph=False)
det.set_source_frames((S, S))
base = np.stack([textured_frame(8100 + s, S, S, n_rect=1200) for s in range(B)])
def T(fn, n=5):
    fn(); torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(n): fn()
    b.record(); torch.cuda.synchronize()
    return a.elapsed_time(b) / n
for name, fr in (("textured", base), ("textured+noise", np.clip(base.astype(np.int16) + np.random.default_rng(1).integers(-40, 41, base.shape), 0, 255).astype(np.uint8)),
                 ("noise", np.random.default_rng(2).integers(0, 256, base.shape, dtype=np.uint8))):
    f0 = torch.from_numpy(fr).to(dev); f1 = torch.from_numpy(np.ascontiguousarray(np.roll(fr, (3, -2), (1, 2)))).to(dev)
    det.src_u8.copy_(f0); det.ingest_u8_launch()
    t_fwd = T(lambda: [fn() for fn, _, _ in det.ops[1:]], 3)
    t_nms = T(lambda: det._nms_launch(True))
    cnt = det.out_count.cpu().numpy()
    gmc = GmcEstimator(B, S, S, 2, max_kp=32768, device=dev)
    gmc.estimate(f0, det.out, det.out_count, det_thresh=0.2)
    k = [0]
    def est():
        k[0] += 1
        gmc.estimate(f1 if k[0] & 1 else f0, det.out, det.out_count, det_thresh=0.2)
    t_gmc = T(est, 4)
    st = gmc.stat.cpu().numpy()
    eng = TrackEngine("botsort", n_seq=B, dtype="f64", cap=1152, dmax=det.max_det, device=dev)
    out = torch.zeros((B, 1152, L.OUT_COLS), dtype=torch.float64, device=dev); stat = torch.zeros((B, L.STAT_WORDS), dtype=torch.int32, device=dev)
    t_trk = T(lambda: eng.step_device(det.out, det.out_count, out, stat, warps=gmc.warps.view(B, 6)), 5)
    print("%-15s fwd %.2f ms  nms %.2f ms (dets %s)  gmc %.2f ms (kp %.0f, inliers %.0f, flags %s)  botsort step %.2f ms (err %d)" % (
        name, t_fwd, t_nms, cnt.tolist(), t_gmc, st[:, 0].mean(), st[:, 4].mean(), sorted(set(st[:, 5].tolist())), t_trk, int(stat[:, L.STAT_ERR].max())))
