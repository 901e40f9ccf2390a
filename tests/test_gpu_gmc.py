"""-m gpu: the camera-motion estimator (csrc/b2t_gmc.cu, SURVEY.md 8f row 1) on an H100 through the C ABI against oracle/gmc.py
(pinned against cv2 and the reference's GMC class by tests/test_oracle_gmc.py): full-size frames, several sequences per call,
detection masks, rotated / scaled motion, the drop-in ``botsort.GMC`` and ``BoTSORT(use_GMC=True)``, the pipelined two-call form."""
import os
import sys

import numpy as np
import pytest

pytestmark = pytest.mark.gpu
torch = pytest.importorskip("torch")

from b200track import _lib as L  # noqa: E402
from b200track.gmc import GmcEstimator  # noqa: E402
from b200track.synth import make_stream, textured_frame  # noqa: E402
from oracle import gmc as OG  # noqa: E402
from oracle import trackers as T  # noqa: E402


def _moved(frame, angle_deg, scale, tx, ty):
    cv2 = pytest.importorskip("cv2")
    h, w = frame.shape[:2]
    M = cv2.getRotationMatrix2D((w / 2, h / 2), angle_deg, scale)
    M[:, 2] += (tx, ty)
    return cv2.warpAffine(frame, M, (w, h), flags=cv2.INTER_LINEAR, borderMode=cv2.BORDER_REFLECT_101)


def _dets(seed, n, h, w):
    """n integer-rounded tlbr boxes with scores in descending order (what the NMS stage hands over)."""
    rng = np.random.default_rng(seed)
    x1 = rng.uniform(0, w - 120, n); y1 = rng.uniform(0, h - 200, n)
    box = np.round(np.stack([x1, y1, x1 + rng.uniform(20, 100, n), y1 + rng.uniform(40, 180, n)], 1))
    score = np.sort(rng.uniform(0.05, 0.95, n))[::-1]
    return np.concatenate([box, score[:, None], rng.integers(0, 3, (n, 1))], 1).astype(np.float32)


@pytest.mark.parametrize("shape", [(720, 1280), (721, 1283)])
def test_stages_bit_exact_vs_oracle(shape):
    h, w = shape
    S = 2
    frames = np.stack([textured_frame(40 + s, h, w, n_rect=900) for s in range(S)])
    dets = np.zeros((S, 32, 6), np.float32)
    cnt = np.array([20, 32], np.int32)
    for s in range(S):
        dets[s, :cnt[s]] = _dets(7 + s, int(cnt[s]), h, w)
    est = GmcEstimator(S, h, w, 2, max_kp=32768)
    warps, stat = est.estimate(torch.from_numpy(frames).cuda(), torch.from_numpy(dets).cuda(), torch.from_numpy(cnt).cuda(), det_thresh=0.2)
    stat = stat.cpu().numpy()
    for s in range(S):
        d = dets[s, :cnt[s]]
        gray, xs, ys, desc = OG.GMCOracle().stages(frames[s], d[d[:, 4] >= np.float32(0.2)])
        kx, ky, kd = est.keypoints(s)
        assert len(xs) > 1000 and stat[s, 0] == len(xs) and not (stat[s, 5] & L.GMC_TRUNCATED)
        assert np.array_equal(kx, xs) and np.array_equal(ky, ys)
        assert np.array_equal(kd, desc)
    assert np.array_equal(warps.cpu().numpy(), np.tile(np.eye(2, 3), (S, 1, 1)))


def test_estimates_vs_oracle_and_cv2_rotating_camera():
    """Three sequences, five frames of rotation + zoom + shift: equal to the restated estimator (same sampling sequence) to 1e-9,
    within OpenCV's own run-to-run spread of cv2.estimateAffinePartial2D, and close to the true motion."""
    h, w, S = 720, 1280, 2
    cur = [textured_frame(60 + s, h, w, n_rect=900) for s in range(S)]
    est = GmcEstimator(S, h, w, 2, max_kp=32768)
    orc = [OG.GMCOracle(estimator="both") for _ in range(S)]          # cv2's estimate returned, the restated one in .last
    rng = np.random.default_rng(3)
    worst_lin = worst_t = 0.0
    for k in range(4):
        warps, stat = est.estimate(torch.from_numpy(np.stack(cur)).cuda())
        warps = warps.cpu().numpy(); stat = stat.cpu().numpy()
        for s in range(S):
            Hr = orc[s].apply(cur[s])
            np.testing.assert_allclose(warps[s], orc[s].last["H_restated"], rtol=0, atol=1e-9)
            if k:
                assert stat[s, 3] == len(orc[s].last["src"]) and stat[s, 4] > 100
                worst_lin = max(worst_lin, float(np.abs(warps[s, :, :2] - Hr[:, :2]).max()))
                worst_t = max(worst_t, float(np.abs(warps[s, :, 2] - Hr[:, 2]).max()))
        cur = [_moved(f, float(rng.uniform(-0.6, 0.6)), 1.0 + float(rng.uniform(-0.004, 0.004)), float(rng.uniform(-8, 8)), float(rng.uniform(-8, 8))) for f in cur]
    print("GPU estimator vs cv2.estimateAffinePartial2D: max |d linear| %.2e, max |d translation| %.3f px" % (worst_lin, worst_t))
    assert worst_lin < 1e-3 and worst_t < 0.25


def test_prepared_two_call_form_equals_single_call():
    h, w, S = 384, 640, 2
    a = [textured_frame(80 + s, h, w) for s in range(S)]
    e1, e2 = GmcEstimator(S, h, w), GmcEstimator(S, h, w)
    for k in range(3):
        fr = torch.from_numpy(np.stack([np.roll(f, (2 * k, -3 * k), (0, 1)) for f in a])).cuda()
        w1, _ = e1.estimate(fr)
        e2.prepare(fr, k & 1)
        w2, _ = e2.estimate_prepared(k & 1)
        assert torch.equal(w1, w2)
    assert float((w1[:, 0, 2] + 3).abs().max()) < 0.5 and float((w1[:, 1, 2] - 2).abs().max()) < 0.5      # the true shift (a rolled frame wraps around: outliers)


def test_dropin_botsort_gmc_and_tracker():
    """tracker/botsort.py surface: GMC(method='orb').apply on host frames equals the oracle's recipe; BoTSORT(use_GMC=True).update
    consumes it -- ids equal to the oracle tracker fed with the same (GPU-estimated) warps."""
    sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "yolov7-tracker_b200", "tracker"))
    import basetrack
    import botsort as B
    from oracle.refshim import Opts
    basetrack.BaseTrack._count = 0
    h = w = 640
    base = textured_frame(90, h, w, n_rect=600)
    frames_d, _ = make_stream(17, 12, n_obj=60, img=w)
    gmc = B.GMC(method='orb', downscale=2)
    orc = OG.GMCOracle(estimator="restated")
    trk = B.BoTSORT(Opts(kalman_format="botsort"), frame_rate=30)
    ot = T.TrackerOracle("botsort")
    for k, d in enumerate(frames_d):
        img = np.ascontiguousarray(np.roll(base, (3 * k, -2 * k), (0, 1)))
        hi = d[d[:, 4] >= np.float32(0.2)]
        H = gmc.apply(img, hi)
        np.testing.assert_allclose(H, orc.apply(img, hi), rtol=0, atol=1e-9)
        out = trk.update(torch.from_numpy(d), torch.from_numpy(img))
        exp = ot.update(d, warp=H)
        assert sorted(int(t.track_id) for t in out) == sorted(e[0] for e in exp)
    assert abs(H[0, 2] + 2) < 0.5 and abs(H[1, 2] - 3) < 0.5


def test_pipeline_botsort_with_gpu_gmc_equals_stepwise():
    """TrackingPipeline(detector, BoT-SORT engine, gmc=estimator): frames in, tracks out, the warp estimated on the device between
    NMS and the tracker step (prepare on the detect stream while the frame buffer is valid, estimate on the tracker stream) --
    the same rows as detect -> estimate -> step done one after the other on one stream."""
    from b200track.detector import DetectorW6
    from b200track.engine import TrackEngine
    from b200track.pipeline import TrackingPipeline
    from b200track.w6 import calibrated_state_dict
    sd = calibrated_state_dict(0, 256, "cuda")
    S, n = 2, 5
    base = np.stack([textured_frame(120 + s, 256, 256, n_rect=300) for s in range(S)])
    frames = [torch.from_numpy(np.ascontiguousarray(np.roll(base, (2 * k, -k), axis=(1, 2)))).pin_memory() for k in range(n)]

    def build():
        det = DetectorW6(sd, batch=S, img_size=256, use_graph=False, autotune=False)
        det.set_source_frames((256, 256))
        return det, TrackEngine("botsort", n_seq=S, cap=1152, dmax=300), GmcEstimator(S, 256, 256, 2, max_kp=4096)      # BoT-SORT births from every first-stage leftover (q3): 5 frames of 300 detections need > 512 slots
    det, eng, gmc = build()
    pipe = TrackingPipeline(det, eng, out_rows=1152, gmc=gmc)
    got = []
    for f in frames:
        r = pipe.step(f)
        if r is not None:
            got.append([r[0][s, :int(r[1][s, L.STAT_NOUT])].clone() for s in range(S)])
    r = pipe.flush()
    got.append([r[0][s, :int(r[1][s, L.STAT_NOUT])].clone() for s in range(S)])
    warps_pipe = gmc.warps.cpu().numpy().copy()
    # ---- the same, step by step on the current stream
    det, eng, gmc = build()
    out = torch.zeros((S, 1152, L.OUT_COLS), dtype=torch.float64, device="cuda")
    stat = torch.zeros((S, L.STAT_WORDS), dtype=torch.int32, device="cuda")
    exp = []
    for f in frames:
        det.src_u8.copy_(f)
        det.ingest_u8_launch()
        for fn, _, _ in det.ops[1:]:                     # ops[0] is the ReOrg of the float tensor, replaced by the uint8 ingest
            fn()
        det._nms_launch(True)
        w, _ = gmc.estimate(det.src_u8, det.out, det.out_count, det_thresh=float(eng.cfg.conf_thresh))
        eng.step_device(det.out, det.out_count, out, stat, warps=w.view(S, 6))
        torch.cuda.synchronize()
        exp.append([out[s, :int(stat[s, L.STAT_NOUT])].cpu().clone() for s in range(S)])
    assert len(got) == len(exp) == n
    rows = 0
    for a, b in zip(got, exp):
        for s in range(S):
            assert a[s].shape == b[s].shape and torch.allclose(a[s], b[s], rtol=0, atol=0, equal_nan=True)
            rows += a[s].shape[0]
    assert rows > 0
    np.testing.assert_array_equal(warps_pipe, gmc.warps.cpu().numpy())
    assert np.isfinite(warps_pipe).all() and np.abs(warps_pipe[:, :, 2]).max() < 8       # (128 x 128 working pixels, 300 boxes masked out: too few points for a precise shift)


def test_gpu_vs_committed_reference_golden():
    """tests/golden/gmc.npz: the matrices of the UNMODIFIED reference GMC class over two seeded sequences (one of odd size) with masked
    detections; the GPU estimate moves the frame's corners by less than a pixel differently (the spread of two RANSAC realisations)."""
    sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden"))
    from make_golden_gmc import CASES, frames_and_dets
    gold = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "gmc.npz"))
    for k, case in enumerate(CASES):
        frames, dets = frames_and_dets(case)
        est = GmcEstimator(1, case["h"], case["w"], 2, max_kp=8192)
        d = torch.from_numpy(dets[None].copy()).cuda()
        for i, f in enumerate(frames):
            w, _ = est.estimate(torch.from_numpy(f[None]).cuda(), d, None, det_thresh=float("-inf"))
            assert OG.corner_displacement(w[0].cpu().numpy(), gold["H%d" % k][i], case["h"], case["w"]) < 1.0, (k, i)
