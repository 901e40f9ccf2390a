"""Writes tests/golden/loop_uavmot.npz: the UNMODIFIED reference ``UAVMOT`` (tracker/uavmot.py).

Run in a checkout next to the reference tree (``python tests/golden/make_golden_uavmot.py``; oracle/refshim.py finds it,
B2T_REFERENCE_ROOT points elsewhere).  ``reid_models.deepsort_reid.Extractor`` is stubbed (the reference builds it and never uses it,
uavmot.py:76-77) and ``matching.linear_assignment`` is wrapped to record every cost matrix with its threshold.
Before anything is written, the oracle (tests/uavmot_oracle.py) must agree with the reference frame by frame, and the stream must
contain: frames where the structure term changes association 1's matching against the IoU cost at 0.8 / 0.98 (the duplicates
uavmot_golden.CONFIGS places for it); a frame where q20 skips
the fused solve (single match (0, 0)); q21 marking an updated track lost; ties of the maximum and of the minimum neighbour length;
lengths on and just inside 400; axis and diagonal neighbour directions; isolated and single-neighbour points.  No cost may lie within
1e-9 of its threshold (0.7 / 0.8 / 0.5), no duplicate distance within 1e-9 of 0.15, no non-tied length within 1e-9 (relative) of
another, no angle within 1e-9 of an integer off the multiples of 45 degrees.
Stored per configuration: per frame the output ids and tlwh (float64) and the tracked and lost lists (id, state, is_activated,
start_frame, frame_id, tracklet_len)."""
import importlib
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
from uavmot_oracle import UavmotOracle                              # noqa: E402
import uavmot_golden as UG                                          # noqa: E402

EPS = 1e-9


def load_uavmot(ref):
    class _Extractor:
        def __init__(self, *a, **k):
            pass

    rm = types.ModuleType("reid_models")
    ds = types.ModuleType("reid_models.deepsort_reid")
    ds.Extractor = _Extractor
    mods = {"basetrack": ref.basetrack, "matching": ref.matching, "kalman_filter": ref.kalman_filter, "reid_models": rm,
            "reid_models.deepsort_reid": ds}
    saved = {k: sys.modules.get(k) for k in list(mods) + ["uavmot"]}
    sys.modules.update(mods)
    tdir = os.path.join(refshim.REF_ROOT, "tracker")
    sys.path.insert(0, tdir)
    try:
        mod = importlib.import_module("uavmot")
    finally:
        sys.path.remove(tdir)
        for k, v in saved.items():
            if v is None:
                sys.modules.pop(k, None)
            else:
                sys.modules[k] = v
    return mod


def run(um, ref, cfg, frames):
    ref.basetrack.BaseTrack._count = 0
    opts = refshim.Opts(kalman_format=cfg.fmt, track_buffer=cfg.track_buffer)
    trk = um.UAVMOT(opts, frame_rate=30)
    m = um.matching
    la, iou_fn, fuse = m.linear_assignment, m.iou_distance, m.local_relation_fuse_motion
    costs, dup, fused = [], [], []

    def la_rec(cost, thresh):
        costs.append((np.array(cost, np.float64), thresh))
        return la(cost, thresh)

    def fuse_rec(*a, **k):
        fused.append(len(costs))
        return fuse(*a, **k)

    rds = um.remove_duplicate_stracks

    def rds_rec(a, b):
        dup.append(np.array(iou_fn(a, b), np.float64))
        return rds(a, b)

    m.linear_assignment, m.local_relation_fuse_motion, um.remove_duplicate_stracks = la_rec, fuse_rec, rds_rec
    img = np.zeros((4, 4, 3), np.uint8)
    out = []
    try:
        for fr in frames:
            cur = trk.update(fr.copy(), img)
            lists = {w: np.array([[t.track_id, t.state, int(t.is_activated), t.start_frame, t.frame_id, t.tracklet_len] for t in L],
                                 np.int64).reshape(-1, 6) for w, L in (("tracked", trk.tracked_stracks), ("lost", trk.lost_stracks))}
            out.append((np.array([t.track_id for t in cur], np.int32), np.array([np.asarray(t.tlwh, np.float64) for t in cur]).reshape(-1, 4),
                        lists))
    finally:
        m.linear_assignment, m.local_relation_fuse_motion, um.remove_duplicate_stracks = la, fuse, rds
    return out, costs, dup, fused


def main():
    ref = refshim.load()
    um = load_uavmot(ref)
    out = dict(ver_numpy=np.__version__, ver_scipy=scipy.__version__)
    for cfg in UG.CONFIGS:
        frames = cfg.stream()
        res, costs, dup, fused = run(um, ref, cfg, frames)
        assert fused, "%s: local_relation_fuse_motion never ran" % cfg.name
        for c, t in costs:
            if c.size:
                assert np.abs(c - t).min() > EPS, "%s: a cost lies at its threshold %.2f" % (cfg.name, t)
        for d in dup:
            if d.size:
                assert np.abs(d - 0.15).min() > EPS, "%s: a duplicate distance lies at 0.15" % cfg.name
        orc = UavmotOracle(kalman_format=cfg.fmt, track_buffer=cfg.track_buffer)
        ev = {}
        for k in range(cfg.n_frames):
            r = orc.update(frames[k])
            assert [t[0] for t in r] == res[k][0].tolist(), "%s frame %d: oracle ids" % (cfg.name, k + 1)
            for e, v in orc.events.items():
                ev[e] = ev.get(e, 0) + v
        info = orc.info
        print("%s: events %s, structure %s" % (cfg.name, ev, info))
        for e in ("s_decides", "q20_skip", "q21_updated"):
            assert ev[e] > 0, "%s: the stream has no %s event" % (cfg.name, e)
        for e in ("tie_max", "tie_min", "on400", "inside400", "axis", "diag", "isolated", "single"):
            assert info.get(e, 0) > 0, "%s: the structure vectors show no %s case" % (cfg.name, e)
        assert info["len_gap"] > EPS and info["angle_gap"] > EPS and info.get("near400", 0) == 0, \
            "%s: a length or angle margin below 1e-9" % cfg.name
        p = cfg.name + "/"
        out.update({p + "digest": UG.stream_digest(frames), p + "count": np.array([len(r[0]) for r in res], np.int32),
                    p + "ids": np.concatenate([r[0] for r in res]), p + "tlwh": np.concatenate([r[1] for r in res])})
        for w in ("tracked", "lost"):
            out[p + w + "_count"] = np.array([len(r[2][w]) for r in res], np.int32)
            out[p + w] = np.concatenate([r[2][w] for r in res])
    np.savez_compressed(UG.PATH, **out)


if __name__ == "__main__":
    main()
