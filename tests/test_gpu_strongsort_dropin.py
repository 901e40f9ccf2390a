"""-m gpu: StrongSORT as track.py reaches it, on an H100.
  * the drop-in ``tracker/strongsort.py``: the body of tracker/track.py:138-179 with ``StrongSORT(opts, gamma=opts.gamma)`` on a synthetic
    720p video, seeded OSNet weights loaded by ``load_pretrained_weights`` and the real ECC estimator, against the oracle fed with the
    features and warps the device computed (read back);
  * ``TrackingPipeline`` with a StrongSORT engine, an ``OsnetExtractor`` and an ``EccEstimator``: B = 4 sequences bit-identical to the
    same sequences through the drop-in one by one; a negative crop raises B2TError naming its sequence; mismatched pairs are refused."""
import os
import sys

import numpy as np
import pytest

pytestmark = pytest.mark.gpu
torch = pytest.importorskip("torch")

HERE = os.path.dirname(os.path.abspath(__file__))
PKG = os.path.join(os.path.dirname(HERE), "yolov7-tracker_b200")
sys.path.insert(0, HERE)
from b200track import _lib as L                                                                # noqa: E402
from b200track.synth import make_strongsort_stream, textured_frame                             # noqa: E402
from strongsort_oracle import StrongSortOracle                                                 # noqa: E402
from test_gpu_reid_pipeline import _scenario, _detector, _reference_rows, _run_pipeline, _pick_thresh, w6_sd, P  # noqa: E402,F401

BARE = ("basetrack", "botsort", "matching", "kalman_filter", "strongsort", "reid_models", "reid_models.OSNet",
        "reid_models.load_model_tools")


@pytest.fixture(scope="module")
def dropin(tmp_path_factory):
    """the drop-in modules imported by their bare names (as track.py does), and a seeded osnet_x0_25 checkpoint"""
    saved = {k: sys.modules.pop(k) for k in list(sys.modules) if k in BARE}
    sys.path.insert(0, os.path.join(PKG, "tracker"))
    try:
        import strongsort
        from basetrack import BaseTrack
        from reid_models.OSNet import osnet_x0_25
        torch.manual_seed(0)
        net = osnet_x0_25(num_classes=1, pretrained=False)
        with torch.no_grad():
            for name, b in net.named_buffers():
                if name.endswith("running_var"):
                    b.uniform_(0.5, 2.0)
                elif name.endswith("running_mean"):
                    b.normal_(0, 0.1)
        path = str(tmp_path_factory.mktemp("osnet") / "osnet_x0_25.pth")
        torch.save({"state_dict": {"module." + k: v for k, v in net.state_dict().items()}}, path)
        yield strongsort, BaseTrack, path
    finally:
        sys.path.remove(os.path.join(PKG, "tracker"))
        for k in BARE:
            sys.modules.pop(k, None)
        sys.modules.update(saved)


class Opts:
    def __init__(self, path, conf_thresh=0.2):
        self.conf_thresh, self.track_buffer, self.kalman_format, self.img_size = conf_thresh, 30, "strongsort", 1280
        self.iou_thresh, self.reid_model_path, self.dhn_path, self.gamma, self.min_area = 0.5, path, "", 0.1, 10


def _record(trk):
    """wrap get_feature / ECC.apply to keep what the device computed"""
    rec = {"feats": None, "warp": None}
    gf, ap = trk.get_feature, trk.ECC.apply

    def get_feature(tlbrs, img):
        f = gf(tlbrs, img)
        rec["feats"] = f.detach().cpu().numpy().copy()
        return f

    def apply(raw_frame, detections=None):
        w = ap(raw_frame, detections)
        rec["warp"] = np.asarray(w, np.float64).copy()
        return w
    trk.get_feature, trk.ECC.apply = get_feature, apply
    return rec


def test_dropin_track_py_body_matches_oracle(dropin):
    strongsort, BaseTrack, path = dropin
    n = 40
    frames, _, _ = make_strongsort_stream(21, n, 30, 64, img=720)
    base = textured_frame(5, 720, 1400, n_rect=400)
    opts = Opts(path)
    BaseTrack._count = 0
    tracker = strongsort.StrongSORT(opts, frame_rate=30, gamma=opts.gamma)
    rec = _record(tracker)
    orc = StrongSortOracle(gamma=opts.gamma)
    results, outputs, moved = [], 0, 0.0
    for i in range(n):
        img0 = np.ascontiguousarray(base[:, 2 * i: 2 * i + 1280])                  # a 1280 x 720 video panning 2 px per frame
        out = frames[i].copy()
        rec["feats"] = None
        current_tracks = tracker.update(out, img0)                                 # track.py:151
        cur_tlwh, cur_id, cur_cls = [], [], []
        for trk in current_tracks:                                                 # track.py:160-170
            bbox, tid, cls = trk.tlwh, trk.track_id, trk.cls
            if bbox[2] * bbox[3] > opts.min_area:
                cur_tlwh.append(bbox); cur_id.append(tid); cur_cls.append(cls)
        results.append((i + 1, cur_id, cur_tlwh, cur_cls))
        sel = out[:, 4] > np.float32(opts.conf_thresh)
        feats = np.zeros((len(out), 512), np.float32)
        if sel.any():
            feats[sel] = rec["feats"]
        exp = orc.update(out, feats, rec["warp"])
        assert [int(t.track_id) for t in current_tracks] == [t[0] for t in exp], "frame %d" % (i + 1)
        np.testing.assert_allclose(np.array([t.tlwh for t in current_tracks]).reshape(-1, 4),
                                   np.array([t[1] for t in exp]).reshape(-1, 4), rtol=0, atol=1e-9)
        if len(current_tracks):
            np.testing.assert_allclose(np.array([t.features[-1] for t in current_tracks]), orc.last_features(), rtol=0, atol=1e-6)
        outputs += len(current_tracks)
        moved = max(moved, abs(rec["warp"][0, 2]))
    assert outputs > 0 and moved > 0.5, (outputs, moved)


def _ss_engine(S, dmax, thr, use_gmc=True):
    # StrongSORT never loses an unmatched Tracked track (q18): on the detector's noise stream the tracked list grows every frame, so
    # the pipeline test runs few frames
    from b200track.engine import TrackEngine
    return TrackEngine("strongsort", n_seq=S, cap=1152, dmax=dmax, feat_dim=512, conf_thresh=thr, use_gmc=use_gmc)


def test_pipeline_strongsort_equals_dropin_per_sequence(w6_sd, dropin):
    from b200track.pipeline import TrackingPipeline
    from b200track.gmc import EccEstimator
    strongsort, BaseTrack, path = dropin
    S, hw = 4, (256, 256)
    frames = _scenario(S, n=5, hw=hw)
    det = _detector(w6_sd, S, hw, hw)
    thr = _pick_thresh(det, frames)
    opts = Opts(path, conf_thresh=thr)
    ref = strongsort.StrongSORT(opts, gamma=0.1)                                   # the drop-in's OSNet with the loaded weights
    ext = ref.reid_model.extractor(torch.device("cuda", torch.cuda.current_device()), (128, 256))
    pipe = TrackingPipeline(det, _ss_engine(S, det.max_det, thr), out_rows=1152, reid=ext, gmc=EccEstimator(S, hw[0], hw[1], 2),
                            reid_cap=S * det.max_det)
    cut = pipe.reid_net.cut

    def widened_cut(fr, d, cnt, t):
        P.widen_degenerate(d, hw)
        return cut(fr, d, cnt, t)
    pipe.reid_net.cut = widened_cut
    got = _run_pipeline(pipe, frames, S)
    dets = []
    d2 = _detector(w6_sd, S, hw, hw)
    for f in frames:
        rows, cnt = _reference_rows(d2, f)
        P.widen_degenerate(rows, hw)
        torch.cuda.synchronize()
        r, c = rows.cpu().numpy(), cnt.cpu().numpy()
        dets.append([r[s, :c[s]].copy() for s in range(S)])
    compared = 0
    for s in range(S):
        BaseTrack._count = 0
        trk = strongsort.StrongSORT(opts, gamma=0.1)
        for k, f in enumerate(frames):
            out = trk.update(dets[k][s].copy(), f[s].numpy())
            mine = got[k][s].numpy()
            assert [int(t.track_id) for t in out] == mine[:, 0].astype(np.int64).tolist(), "frame %d sequence %d" % (k, s)
            assert np.array_equal(np.array([t.tlwh for t in out]).reshape(-1, 4), mine[:, 1:5]), "frame %d sequence %d" % (k, s)
            compared += len(out)
    assert compared > 0


def test_pipeline_strongsort_errors(w6_sd, dropin):
    from b200track.pipeline import TrackingPipeline
    from b200track.gmc import EccEstimator, GmcEstimator
    strongsort, BaseTrack, path = dropin
    S, hw = 4, (256, 256)
    ext = strongsort.StrongSORT(Opts(path), gamma=0.1).reid_model.extractor(torch.device("cuda", torch.cuda.current_device()), (128, 256))
    det = _detector(w6_sd, S, hw, hw)
    from b200track.engine import TrackEngine
    bot = TrackEngine("botsort", n_seq=S, cap=1152, dmax=det.max_det, feat_dim=512)
    with pytest.raises(L.B2TError, match="StrongSORT engine"):
        TrackingPipeline(det, bot, reid=ext)
    with pytest.raises(L.B2TError, match="OsnetExtractor"):
        TrackingPipeline(det, _ss_engine(S, det.max_det, 0.05), reid=object())        # e.g. a ReidExtractor
    with pytest.raises(L.B2TError, match="EccEstimator"):
        TrackingPipeline(det, _ss_engine(S, det.max_det, 0.05), reid=ext, gmc=GmcEstimator(S, hw[0], hw[1]))
    with pytest.raises(L.B2TError, match="GmcEstimator"):
        TrackingPipeline(det, TrackEngine("botsort", n_seq=S, cap=1152, dmax=det.max_det), gmc=EccEstimator(S, hw[0], hw[1]))
    # a negative crop in sequence 2 raises when the step's tracks are collected
    pipe = TrackingPipeline(det, _ss_engine(S, det.max_det, 0.05), out_rows=1152, reid=ext, gmc=None)
    cut = pipe.reid_net.cut

    def bad_cut(fr, d, cnt, t):
        P.widen_degenerate(d, hw)
        d[2, 0, :5] = torch.tensor([-6.0, -6.0, 20.0, 20.0, 0.9], device=d.device)
        cnt[2] = torch.clamp(cnt[2], min=1)
        return cut(fr, d, cnt, t)
    pipe.reid_net.cut = bad_cut
    frames = _scenario(S, n=2, hw=hw)
    with pytest.raises(L.B2TError, match="sequence 2"):
        for f in frames:
            pipe.step(f)
        pipe.flush()
