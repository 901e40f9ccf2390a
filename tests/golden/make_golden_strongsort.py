"""Writes tests/golden/loop_strongsort.npz: the UNMODIFIED reference ``StrongSORT`` (tracker/strongsort.py).

Run in a checkout next to the reference tree (``python tests/golden/make_golden_strongsort.py``; oracle/refshim.py finds it,
B2T_REFERENCE_ROOT points elsewhere).  The reference runs as shipped; the stand-ins live here, not in the shared refshim:
  * ``reid_models.OSNet.osnet_x0_25`` / ``.cuda()`` / ``load_pretrained_weights``: stubs (no network, no checkpoint);
  * ``tracker.get_feature``: returns the stream's stored float32 feature rows, and checks that it is called once per frame with
    exactly the ``score > det_thresh`` rows;
  * ``tracker.ECC`` = refshim.FixedGMC with the stream's float32 warps (stored as float64);
  * ``matching.linear_assignment`` wrapped to record every cost matrix with its threshold.
Before anything is written, the stream is checked (with the oracle, tests/strongsort_oracle.py, which must agree with the reference
frame by frame) for: ids that differ from the same stream at gamma = 1; association-1 matches at zero IoU, one of them a Lost track
re-activated across a jump; q18 marking an updated track lost and an unmatched Tracked track coasting; an unconfirmed track matched
at zero IoU in association 3; and no assignment cost within 1e-9 of its threshold (0.7 / 0.5), no duplicate distance within 1e-9 of
0.15.
Stored per configuration: per frame the output ids and tlwh (float64), the tracked and lost lists (id, state, is_activated,
start_frame, frame_id, tracklet_len), and every 8th frame the features (track.features[-1]) of the output tracks."""
import os
import sys
import types

import numpy as np
import scipy

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, os.path.join(ROOT, "yolov7-tracker_b200"))

from oracle import refshim                                          # noqa: E402
from b200track.synth import stream_digest                           # noqa: E402
from strongsort_oracle import StrongSortOracle                      # noqa: E402
import strongsort_golden as SG                                      # noqa: E402

EPS = 1e-9


def load_strongsort(ref):
    """Imports the reference's strongsort.py against the modules refshim loaded, with the OSNet constructor and loader stubbed."""
    class _Net:
        def cuda(self):
            return self

        def eval(self):
            return self

    mods = {"basetrack": ref.basetrack, "matching": ref.matching, "botsort": ref.botsort, "kalman_filter": ref.kalman_filter}
    rm = types.ModuleType("reid_models")
    osn = types.ModuleType("reid_models.OSNet")
    osn.osnet_x0_25 = lambda *a, **k: _Net()
    lmt = types.ModuleType("reid_models.load_model_tools")
    lmt.load_pretrained_weights = lambda model, path: None
    mods.update({"reid_models": rm, "reid_models.OSNet": osn, "reid_models.load_model_tools": lmt})
    saved = {k: sys.modules.get(k) for k in list(mods) + ["strongsort"]}
    sys.modules.update(mods)
    tdir = os.path.join(refshim.REF_ROOT, "tracker")
    sys.path.insert(0, tdir)
    try:
        import importlib
        mod = importlib.import_module("strongsort")
    finally:
        sys.path.remove(tdir)
        for k, v in saved.items():
            if v is None:
                sys.modules.pop(k, None)
            else:
                sys.modules[k] = v
    return mod


class StoredFeatures:
    """get_feature stand-in: the stored features of the frame's score > det_thresh rows, in row order."""

    def __init__(self, frames, feats, det_thresh):
        self.frames, self.feats, self.det_thresh = frames, feats, det_thresh
        self.k, self.calls = -1, 0

    def __call__(self, tlbrs, ori_img):
        sel = self.frames[self.k][:, 4] > self.det_thresh
        assert np.array_equal(np.asarray(tlbrs), self.frames[self.k][sel, :4]), "frame %d: get_feature rows" % self.k
        self.calls += 1
        return self.feats[self.k][sel].copy()


def run(ss, ref, cfg, frames, feats, warps, gamma):
    ref.basetrack.BaseTrack._count = 0
    opts = refshim.Opts(kalman_format=cfg.fmt, track_buffer=cfg.track_buffer)
    trk = ss.StrongSORT(opts, frame_rate=30, gamma=gamma, use_ECC=cfg.use_ecc)
    trk.ECC = refshim.FixedGMC(warps)
    stub = StoredFeatures(frames, feats, trk.det_thresh)
    trk.get_feature = stub
    m = ss.matching
    la, iou_fn = m.linear_assignment, m.iou_distance
    costs, dup = [], []

    def la_rec(cost, thresh):
        costs.append((np.array(cost, np.float64), thresh))
        return la(cost, thresh)

    rds = ss.remove_duplicate_stracks

    def rds_rec(a, b):
        dup.append(np.array(iou_fn(a, b), np.float64))
        return rds(a, b)

    m.linear_assignment, ss.remove_duplicate_stracks = la_rec, rds_rec
    img = np.zeros((4, 4, 3), np.uint8)
    out = []
    try:
        for k, fr in enumerate(frames):
            stub.k = k
            calls = stub.calls
            cur = trk.update(fr.copy(), img)
            assert stub.calls == calls + int((fr[:, 4] > trk.det_thresh).any()), "frame %d: one get_feature call expected" % k
            lists = {w: np.array([[t.track_id, t.state, int(t.is_activated), t.start_frame, t.frame_id, t.tracklet_len] for t in L],
                                 np.int64).reshape(-1, 6) for w, L in (("tracked", trk.tracked_stracks), ("lost", trk.lost_stracks))}
            out.append((np.array([t.track_id for t in cur], np.int32),
                        np.array([np.asarray(t.tlwh, np.float64) for t in cur]).reshape(-1, 4),
                        np.array([t.features[-1] for t in cur], np.float32).reshape(len(cur), -1), lists))
    finally:
        m.linear_assignment, ss.remove_duplicate_stracks = la, rds
    return out, costs, dup


def main():
    ref = refshim.load()
    ss = load_strongsort(ref)
    out = dict(ver_numpy=np.__version__, ver_scipy=scipy.__version__)
    for cfg in SG.CONFIGS:
        frames, feats, warps = cfg.stream()
        res, costs, dup = run(ss, ref, cfg, frames, feats, warps, cfg.gamma)
        g1, _, _ = run(ss, ref, cfg, frames, feats, warps, 1.0)
        differ = [k for k in range(cfg.n_frames) if not np.array_equal(res[k][0], g1[k][0])]
        assert differ, "%s: appearance changes no track id" % cfg.name
        for c, t in costs:
            if c.size:
                assert np.abs(c - t).min() > EPS, "%s: a cost lies at its threshold %.2f" % (cfg.name, t)
        for d in dup:
            if d.size:
                assert np.abs(d - 0.15).min() > EPS, "%s: a duplicate distance lies at 0.15" % cfg.name
        # the oracle agrees frame by frame, and reports the events the stream must contain
        orc = StrongSortOracle(gamma=cfg.gamma, use_ecc=cfg.use_ecc, kalman_format=cfg.fmt, track_buffer=cfg.track_buffer)
        ev = {}
        for k in range(cfg.n_frames):
            r = orc.update(frames[k], feats[k], warps[k] if cfg.use_ecc else None)
            assert [t[0] for t in r] == res[k][0].tolist(), "%s frame %d: oracle ids" % (cfg.name, k + 1)
            for e, v in orc.events.items():
                ev[e] = ev.get(e, 0) + v
        for e in ("zero_iou1", "zero_iou_react1", "q18_updated", "coast", "zero_iou3"):
            assert ev[e] > 0, "%s: the stream has no %s event" % (cfg.name, e)
        keep = [i for i in range(cfg.n_frames) if i % 8 == 7 or i == cfg.n_frames - 1]
        p = cfg.name + "/"
        out.update({p + "digest": stream_digest(frames), p + "feat_digest": stream_digest(feats),
                    p + "count": np.array([len(r[0]) for r in res], np.int32), p + "ids": np.concatenate([r[0] for r in res]),
                    p + "tlwh": np.concatenate([r[1] for r in res]), p + "feat_frames": np.array(keep, np.int32),
                    p + "feats": np.concatenate([res[i][2] for i in keep]),
                    p + "frames_differ": np.array(differ, np.int32)})
        for w in ("tracked", "lost"):
            out[p + w + "_count"] = np.array([len(r[3][w]) for r in res], np.int32)
            out[p + w] = np.concatenate([r[3][w] for r in res])
        print("%s: %d frames, max id %d, ids differ from gamma = 1 on %d frames, events %s"
              % (cfg.name, cfg.n_frames, out[p + "ids"].max(), len(differ), ev))
    np.savez_compressed(os.path.join(HERE, "loop_strongsort.npz"), **out)


if __name__ == "__main__":
    main()
