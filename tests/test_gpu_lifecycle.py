"""-m gpu: the nvcc-built fused tracker step on an H100 against the reference's track life cycle (tests/golden/loop_lifecycle.npz,
written from the unmodified reference by tests/golden/make_golden_lifecycle.py) and against the oracle: every tracker kind with
every Kalman format, non-default options, long-lost pruning, duplicate removal, empty frames, threshold ties, slot recycling, the
float32 build, lap_solve in float32, and the drop-in modules' tracked / lost / removed lists.  Nothing here reads the reference tree."""
import os
import sys

import numpy as np
import pytest

pytestmark = pytest.mark.gpu
torch = pytest.importorskip("torch")

from b200track import _lib as L                         # noqa: E402
from b200track.synth import lifecycle_stream            # noqa: E402
from oracle import lapjv as olap, iou as oiou, trackers as T   # noqa: E402
import lifecycle_golden as LG                           # noqa: E402

CONFIGS = LG.configs()
PKG = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "yolov7-tracker_b200")


def _engine(cfg, **kw):
    from b200track.engine import TrackEngine
    return TrackEngine(cfg.kind, kalman_format=cfg.fmt, conf_thresh=cfg.conf_thresh, track_buffer=cfg.track_buffer,
                       frame_rate=cfg.frame_rate, **kw)


def _int_rows(rows):
    """b2t_tracker_read_list rows -> id, state, is_activated, start_frame, frame_id, tracklet_len (the golden's columns)."""
    return rows[:, [0, 8, 9, 11, 12, 10]].astype(np.int64)


def _maxdiff(a, b):
    return float(np.abs(np.asarray(a) - np.asarray(b)).max(initial=0.0))


@pytest.mark.parametrize("name", CONFIGS)
def test_fused_step_lifecycle_matches_reference(name):
    cfg = LG.Config(name)
    frames, warps = cfg.stream()
    eng = _engine(cfg, cap=256, dmax=128)
    worst = 0.0
    for i in range(cfg.n_frames):
        where = "%s frame %d" % (name, i + 1)
        got = eng.step([frames[i]], warps=None if warps is None else warps[i].reshape(1, 6))[0]
        assert eng.np_stat[0, L.STAT_ERR] == 0, where
        assert got[:, 0].astype(np.int64).tolist() == cfg.out_ids[i].tolist(), where
        assert np.array_equal(got[:, 5].astype(np.float32), cfg.out_cls[i]), where
        for which in ("tracked", "lost"):
            rows = eng.read_list(0, which)
            assert np.array_equal(_int_rows(rows), cfg.rows[which][i]), "%s: %s list" % (where, which)
            if i in cfg.tlwh_frames:
                np.testing.assert_allclose(rows[:, 1:5], cfg.tlwh[(which, i)], rtol=1e-9, atol=1e-9, err_msg=where)
                worst = max(worst, _maxdiff(rows[:, 1:5], cfg.tlwh[(which, i)]))
        if i in cfg.tlwh_frames:
            np.testing.assert_allclose(got[:, 1:5], cfg.tlwh[("out", i)], rtol=1e-9, atol=1e-9, err_msg=where)
            worst = max(worst, _maxdiff(got[:, 1:5], cfg.tlwh[("out", i)]))
    print("\n%s: largest f64 box difference to the reference %.3g px" % (name, worst))


@pytest.mark.parametrize("kind,fmt", [("bytetrack", "default"), ("bytetrack", "strongsort"), ("botsort", "botsort"),
                                      ("botsort", "strongsort")])
def test_fused_step_lifecycle_eight_sequences_against_oracle(kind, fmt):
    """8 sequences x 300 frames in one engine, each with its own seed (so prunings, duplicates and empty frames fall on different
    frames in different CTAs), against one oracle per sequence."""
    from b200track.engine import TrackEngine
    S, F = 8, 300
    streams = [lifecycle_stream(900 + s, F, 40, warp_sigma=2.0 if kind == "botsort" else 0.0) for s in range(S)]
    eng = TrackEngine(kind, n_seq=S, kalman_format=fmt, cap=256, dmax=128)
    orcs = [T.TrackerOracle(kind, kalman_format=fmt) for _ in range(S)]
    worst = 0.0
    for i in range(F):
        warps = np.stack([streams[s][1][i].reshape(6) for s in range(S)]) if kind == "botsort" else None
        got = eng.step([streams[s][0][i] for s in range(S)], warps=warps)
        for s in range(S):
            exp = orcs[s].update(streams[s][0][i], streams[s][1][i] if kind == "botsort" else None)
            assert got[s][:, 0].astype(np.int64).tolist() == [e[0] for e in exp], "seq %d frame %d" % (s, i + 1)
            if exp:
                np.testing.assert_allclose(got[s][:, 1:5], np.array([e[1] for e in exp]), rtol=1e-9, atol=1e-9)
                worst = max(worst, _maxdiff(got[s][:, 1:5], np.array([e[1] for e in exp])))
            assert eng.np_stat[s, L.STAT_NTRACKED] == len(orcs[s].tracked) and eng.np_stat[s, L.STAT_NLOST] == len(orcs[s].lost)
    assert int(eng.np_stat[:, L.STAT_ERR].max()) == 0
    print("\n%s/%s: largest f64 box difference to the oracle %.3g px" % (kind, fmt, worst))


def test_fused_step_recycles_slots():
    """A pool only just larger than the most tracks ever alive at once (plus that frame's births), over 600 frames: every slot is
    freed and reused several times; ids and boxes still equal the oracle's and no capacity error is raised."""
    from b200track.engine import TrackEngine
    frames, _ = lifecycle_stream(700, 600, 80)
    orc = T.TrackerOracle("bytetrack")
    exp, peak, live = [], 0, 0
    for f in frames:
        exp.append(orc.update(f))
        peak = max(peak, live + orc.last_stats["births"])
        live = len(orc.tracked) + len(orc.lost)
    cap = peak + 2
    assert cap >= 64, cap                                    # the engine's smallest pool
    eng = TrackEngine("bytetrack", cap=cap, dmax=128)
    for i, f in enumerate(frames):
        got = eng.step([f])[0]
        assert got[:, 0].astype(np.int64).tolist() == [e[0] for e in exp[i]], "frame %d" % (i + 1)
        if exp[i]:
            np.testing.assert_allclose(got[:, 1:5], np.array([e[1] for e in exp[i]]), rtol=1e-9, atol=1e-9)
    assert int(eng.np_stat[0, L.STAT_ERR]) == 0
    assert int(eng.np_stat[0, L.STAT_NEXT_ID]) > 3 * cap, (int(eng.np_stat[0, L.STAT_NEXT_ID]), cap)


@pytest.mark.parametrize("name", CONFIGS)
def test_fused_step_f32_lifecycle(name):
    """The float32 build on the lifecycle streams: the reference's ids on every frame (they agree everywhere on these streams,
    threshold ties included: the scores are compared as float32 in both), boxes within 1e-4 of the float64 reference."""
    cfg = LG.Config(name)
    frames, warps = cfg.stream()
    eng = _engine(cfg, cap=256, dmax=128, dtype="f32")
    for i in range(cfg.n_frames):
        got = eng.step([frames[i]], warps=None if warps is None else warps[i].reshape(1, 6))[0]
        assert got[:, 0].astype(np.int64).tolist() == cfg.out_ids[i].tolist(), "%s frame %d" % (name, i + 1)
        if i in cfg.tlwh_frames:
            np.testing.assert_allclose(got[:, 1:5], cfg.tlwh[("out", i)], rtol=1e-4, atol=2e-2)


@pytest.mark.parametrize("n,m,t", [(1, 1, 0.9), (17, 23, 0.9), (64, 64, 0.5), (150, 120, 0.7), (300, 310, 0.9)])
def test_lap_solve_f32_on_iou_costs(n, m, t):
    """lap_solve in float32 on IoU-distance problems (non-integer boxes, so the optimum is unique): the assignment equals, index
    for index, the float64 optimum of the float32-rounded costs."""
    from b200track.engine import ops as get_ops
    ops = get_ops()
    rng = np.random.default_rng(n * 7 + m)
    a = rng.uniform(0, 500, (n, 2)); a = np.concatenate([a, a + rng.uniform(8, 90, (n, 2))], 1)
    b = a[rng.integers(0, n, m)] + rng.normal(0, 6, (m, 4))
    c32 = (1.0 - oiou.ious(a, b)).astype(np.float32)
    x, y = ops.lap_solve(L.F32, torch.as_tensor(c32, device=ops.device), t)
    _, ex, ey = olap.lapjv(c32.astype(np.float64), True, t)
    assert np.array_equal(x.cpu().numpy(), ex) and np.array_equal(y.cpu().numpy(), ey)


class _Opts:
    def __init__(self, kalman_format, conf_thresh, track_buffer):
        self.conf_thresh, self.track_buffer, self.kalman_format = conf_thresh, track_buffer, kalman_format
        self.img_size, self.iou_thresh, self.reid_model_path, self.dhn_path = 1280, 0.5, "", ""
        self.b2t_cap, self.b2t_dmax = 256, 128


class _FixedGMC:
    def __init__(self, warps):
        self.warps, self.k = warps, 0

    def apply(self, raw_frame=None, detections=None):
        self.k += 1
        return self.warps[self.k - 1]


@pytest.mark.parametrize("name", CONFIGS)
def test_dropin_lists_match_reference(name):
    """BaseTracker / ByteTrack / BoTSORT(opts, frame_rate): every frame, the returned ids, tracked_stracks and lost_stracks (order,
    state, is_activated, start_frame, frame_id, tracklet_len, tlwh) and the removed_stracks appends (ids, order) equal the
    reference's."""
    names = ("basetrack", "bytetrack", "botsort", "matching", "kalman_filter")
    saved = {k: sys.modules.pop(k) for k in names if k in sys.modules}
    sys.path.insert(0, os.path.join(PKG, "tracker"))
    try:
        import basetrack, bytetrack, botsort
        cfg = LG.Config(name)
        frames, warps = cfg.stream()
        opts = _Opts(cfg.fmt, cfg.conf_thresh, cfg.track_buffer)
        basetrack.BaseTrack._count = 0
        if cfg.kind == "sort":
            trk = basetrack.BaseTracker(opts, frame_rate=cfg.frame_rate)
        elif cfg.kind == "bytetrack":
            trk = bytetrack.ByteTrack(opts, frame_rate=cfg.frame_rate)
        else:
            trk = botsort.BoTSORT(opts, frame_rate=cfg.frame_rate)
            trk.gmc = _FixedGMC(warps)
        assert trk.removed_stracks == []                     # start the removed-list bookkeeping at frame 1
        img = np.zeros((4, 4, 3), np.uint8)
        n_removed = 0
        for i, f in enumerate(frames):
            where = "%s frame %d" % (name, i + 1)
            cur = trk.update(f, img)
            assert [t.track_id for t in cur] == cfg.out_ids[i].tolist(), where
            for which, lst in (("tracked", trk.tracked_stracks), ("lost", trk.lost_stracks)):
                rows = np.array([[t.track_id, t.state, int(t.is_activated), t.start_frame, t.frame_id, t.tracklet_len]
                                 for t in lst], np.int64).reshape(-1, 6)
                assert np.array_equal(rows, cfg.rows[which][i]), "%s: %s_stracks" % (where, which)
                if i in cfg.tlwh_frames:
                    np.testing.assert_allclose(np.array([t.tlwh for t in lst]).reshape(-1, 4), cfg.tlwh[(which, i)],
                                               rtol=1e-9, atol=1e-9, err_msg=where)
            removed = trk.removed_stracks
            assert [t.track_id for t in removed[n_removed:]] == cfg.rem_ids[i].tolist(), "%s: removed_stracks" % where
            assert all(t.state == basetrack.TrackState.Removed for t in removed[n_removed:]), where
            n_removed = len(removed)
        assert basetrack.BaseTrack._count == cfg.events["births"]
    finally:
        sys.path.remove(os.path.join(PKG, "tracker"))
        for k in names:
            sys.modules.pop(k, None)
        sys.modules.update(saved)
