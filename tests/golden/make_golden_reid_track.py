"""Writes tests/golden/loop_botsort_reid.npz: the UNMODIFIED reference ``BoTSORT`` with ``use_apperance_model = True``.

Run in a checkout next to the reference tree (``python tests/golden/make_golden_reid_track.py``; oracle/refshim.py imports it,
B2T_REFERENCE_ROOT points elsewhere).  The reference runs as shipped, with three stand-ins:
  * ``tracker.gmc`` = refshim.FixedGMC: the stream's prescribed warps (the role of the reference's own 'file' method);
  * ``tracker.reid_model`` = a stub returning the stream's stored feature rows of the frame's ``det_high`` rows, in row order; it
    checks that it is called once per frame with exactly one crop per ``det_high`` row;
  * ``matching.iou_distance`` / ``matching.embedding_distance`` wrapped to record the costs of associations 1 and 3.
The stream (b200track.synth.make_reid_stream) is checked for two properties before anything is written:
  * the track ids differ from those of the same stream with appearance off on some frames (the feature path decides something);
  * no IoU distance lies within 1e-9 of theta_iou, no appearance cost within 1e-9 of theta_emb and no fused cost within 1e-9 of
    the 0.9 / 0.7 thresholds -- so a different summation order cannot flip a decision.
Stored: the stream configuration and digest, per frame the output track ids and tlwh (float64), and the smoothed features
(track.features[-1], float32) of the output tracks every 8th frame and on the last frame."""
import os
import sys

import numpy as np
import scipy

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "yolov7-tracker_b200"))

from oracle import refshim                                     # noqa: E402
from b200track.synth import make_reid_stream, stream_digest    # noqa: E402

SEED, N_OBJ, N_FRAMES, FEAT_DIM = 32, 60, 80, 64
THETA_IOU, THETA_EMB = 0.5, 0.25
EPS = 1e-9


class StoredFeatures:
    """reid_model stand-in: the features of the current frame's det_high rows."""

    def __init__(self, frames, feats, det_thresh):
        self.frames, self.feats, self.det_thresh = frames, feats, det_thresh
        self.k = -1
        self.calls = 0

    def __call__(self, crops):
        hi = self.frames[self.k][:, 4] >= self.det_thresh
        assert len(crops) == int(hi.sum()), "frame %d: %d crops for %d det_high rows" % (self.k, len(crops), int(hi.sum()))
        self.calls += 1
        return self.feats[self.k][hi].copy()


def run(ref, frames, feats, warps, appearance):
    ref.basetrack.BaseTrack._count = 0
    trk = ref.botsort.BoTSORT(refshim.Opts(kalman_format="botsort"))
    trk.gmc = refshim.FixedGMC(warps)
    trk.use_apperance_model = appearance
    stub = StoredFeatures(frames, feats, trk.det_thresh)
    trk.reid_model = stub
    assert (trk.theta_iou, trk.theta_emb) == (THETA_IOU, THETA_EMB)
    m = ref.botsort.matching
    iou_fn, emb_fn = m.iou_distance, m.embedding_distance
    costs, last_iou = [], []

    def iou_rec(*a, **k):
        r = iou_fn(*a, **k)
        last_iou[:] = [r]
        return r

    def emb_rec(*a, **k):
        r = emb_fn(*a, **k)
        costs.append((last_iou[0].copy(), 0.5 * r))
        return r

    m.iou_distance, m.embedding_distance = iou_rec, emb_rec
    img = np.zeros((4, 4, 3), np.uint8)
    res = []
    try:
        for k, f in enumerate(frames):
            stub.k = k
            calls = stub.calls
            cur = trk.update(f.copy(), img)
            if appearance:
                assert stub.calls == calls + int((f[:, 4] >= trk.det_thresh).any()), "frame %d: one extractor call expected" % k
            res.append((np.array([t.track_id for t in cur], np.int32),
                        np.array([np.asarray(t.tlwh, np.float64) for t in cur]).reshape(-1, 4),
                        np.array([t.features[-1] for t in cur], np.float32).reshape(len(cur), -1) if appearance else None))
    finally:
        m.iou_distance, m.embedding_distance = iou_fn, emb_fn
    return res, costs


def check_margins(costs):
    n_app = 0
    for iou, app in costs:
        if iou.size == 0:
            continue
        assert np.abs(iou - THETA_IOU).min() > EPS, "an IoU distance lies at theta_iou"
        gated = iou <= THETA_IOU
        n_app += int(gated.sum())
        if gated.any():
            assert np.abs(app[gated] - THETA_EMB).min() > EPS, "an appearance cost lies at theta_emb"
        a = app.copy()
        a[iou > THETA_IOU] = 1
        a[a > THETA_EMB] = 1
        dist = np.minimum(iou, a)
        for t in (0.9, 0.7):
            assert np.abs(dist - t).min() > EPS, "a fused cost lies at %.1f" % t
    return n_app


def main():
    ref = refshim.load()
    frames, feats, warps = make_reid_stream(SEED, N_FRAMES, N_OBJ, FEAT_DIM)
    res, costs = run(ref, frames, feats, warps, True)
    off, _ = run(ref, frames, feats, warps, False)
    differ = [k for k in range(N_FRAMES) if not np.array_equal(res[k][0], off[k][0])]
    assert differ, "appearance changes no track id on this stream"
    n_app = check_margins(costs)
    norms = np.linalg.norm(np.concatenate(feats), axis=1)
    assert np.abs(norms - 1).min() > 0.5                      # no detection feature is (close to) a unit vector
    keep = [i for i in range(N_FRAMES) if i % 8 == 7 or i == N_FRAMES - 1]
    out = dict(cfg=np.array([SEED, N_OBJ, N_FRAMES, FEAT_DIM]), digest=stream_digest(frames), feat_digest=stream_digest(feats),
               count=np.array([len(r[0]) for r in res], np.int32), ids=np.concatenate([r[0] for r in res]),
               tlwh=np.concatenate([r[1] for r in res]), feat_frames=np.array(keep, np.int32),
               feats=np.concatenate([res[i][2] for i in keep]), frames_differ=np.array(differ, np.int32),
               ver_numpy=np.__version__, ver_scipy=scipy.__version__)
    np.savez_compressed(os.path.join(HERE, "loop_botsort_reid.npz"), **out)
    print("loop_botsort_reid: %d frames, max id %d, ids differ from IoU-only on %d frames, %d appearance pairs"
          % (N_FRAMES, out["ids"].max(), len(differ), n_app))


if __name__ == "__main__":
    main()
