"""not-gpu: the fused tracker step (csrc/b2t_step.cuh) under the fiber simulator against the reference's track life cycle
(tests/golden/loop_lifecycle.npz): every tracker kind with every Kalman format, non-default conf_thresh / track_buffer /
frame_rate, long-lost pruning, duplicate removal, empty frames and threshold ties.  The tracked and lost lists come from
b2t_tracker_read_list, the removed-list appends from the drop-in's ``removed_in_step`` over the same rows."""
import ctypes as C
import os
import sys

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "hostsim"))
from simlib import ptr, sim, SimTracker  # noqa: E402
from b200track import _lib as L  # noqa: E402
from b200track.synth import lifecycle_stream  # noqa: E402
from oracle import trackers as T  # noqa: E402
import lifecycle_golden as LG  # noqa: E402

CONFIGS = LG.configs()
LIST_COLS = 13


def read_list(trk, which, seq=0):
    """b2t_tracker_read_list rows of one sequence: which = 0 tracked, 1 lost, 2 every slot."""
    lib = sim()
    assert lib.b2t_tracker_list_cols() == LIST_COLS
    rows = np.zeros((trk.cap + 1, LIST_COLS))
    n = C.c_int(-1)
    L.check(lib, lib.b2t_tracker_read_list(trk.h, seq, which, ptr(rows), trk.cap, C.byref(n), None))
    return rows[:n.value].copy()


def _removed_in_step():
    tdir = os.path.join(os.path.dirname(HERE), "yolov7-tracker_b200", "tracker")
    sys.path.insert(0, tdir)
    try:
        import basetrack
    finally:
        sys.path.remove(tdir)
    return basetrack.removed_in_step


def _same_boxes(kind, got, exp, what):
    """Boxes are bit-exact, except under BoT-SORT: the camera-warp products (b2t_gmc_apply) may round the last ulp differently
    from NumPy's R8 @ P @ R8^T, and that carries through the later updates (measured: under 2e-13 px)."""
    if kind == "botsort":
        np.testing.assert_allclose(got, exp, rtol=1e-12, atol=1e-9, err_msg=what)
    else:
        assert np.array_equal(got, exp), what


def _int_rows(rows):
    """list rows -> id, state, is_activated, start_frame, frame_id, tracklet_len (the golden's columns)."""
    return rows[:, [0, 8, 9, 11, 12, 10]].astype(np.int64)


@pytest.mark.parametrize("name", CONFIGS)
def test_fused_step_lifecycle_matches_reference(name):
    cfg = LG.Config(name)
    frames, warps = cfg.stream()
    trk = SimTracker(cfg.kind, kalman_format=cfg.fmt, conf_thresh=cfg.conf_thresh, track_buffer=cfg.track_buffer,
                     frame_rate=cfg.frame_rate, cap=256, dmax=128, ecap=8192)
    removed_in_step = _removed_in_step()
    prev = {0: np.zeros((0, LIST_COLS)), 1: np.zeros((0, LIST_COLS))}
    for i in range(cfg.n_frames):
        where = "%s frame %d" % (name, i + 1)
        res = trk.step([frames[i]], warps=None if warps is None else warps[i].reshape(1, 6))[0]
        assert trk.stat[0, L.STAT_ERR] == 0, where
        assert res[:, 0].astype(np.int64).tolist() == cfg.out_ids[i].tolist(), where
        assert np.array_equal(res[:, 5].astype(np.float32), cfg.out_cls[i]), where
        lists = {w: read_list(trk, w) for w in (0, 1)}
        for w, which in ((0, "tracked"), (1, "lost")):
            assert np.array_equal(_int_rows(lists[w]), cfg.rows[which][i]), "%s: %s list" % (where, which)
            if i in cfg.tlwh_frames:
                _same_boxes(cfg.kind, lists[w][:, 1:5], cfg.tlwh[(which, i)], "%s: %s boxes" % (where, which))
        if i in cfg.tlwh_frames:
            _same_boxes(cfg.kind, res[:, 1:5], cfg.tlwh[("out", i)], where)
        rem = removed_in_step(prev[0], prev[1], read_list(trk, 2), i + 1, cfg.max_time_lost)
        assert [int(r[0]) for r in rem] == cfg.rem_ids[i].tolist(), "%s: removed_stracks appends" % where
        assert all(r[8] == 3 for r in rem), where
        prev = lists


def test_fused_step_lifecycle_three_sequences_against_oracle():
    """One engine, three sequences with different seeds and event timings (ByteTrack, NSA Kalman filter, track_buffer 12): each
    sequence's ids, lists and boxes equal its own oracle's, frame by frame."""
    seeds, n_frames = (501, 502, 503), 80
    streams = [lifecycle_stream(s, n_frames, 30, conf_thresh=0.3)[0] for s in seeds]
    kw = dict(conf_thresh=0.3, track_buffer=12, frame_rate=30)
    trk = SimTracker("bytetrack", kalman_format="strongsort", n_seq=3, cap=192, dmax=96, ecap=4096, **kw)
    orcs = [T.TrackerOracle("bytetrack", kalman_format="strongsort", **kw) for _ in seeds]
    for i in range(n_frames):
        res = trk.step([s[i] for s in streams])
        for q, orc in enumerate(orcs):
            exp = orc.update(streams[q][i])
            where = "sequence %d frame %d" % (q, i + 1)
            assert res[q][:, 0].astype(np.int64).tolist() == [e[0] for e in exp], where
            if exp:
                assert np.array_equal(res[q][:, 1:5], np.array([e[1] for e in exp])), where
            for w, which in ((0, "tracked"), (1, "lost")):
                rows, tlwh = orc.list_rows(which)
                got = read_list(trk, w, q)
                assert np.array_equal(_int_rows(got), rows), "%s: %s list" % (where, which)
                assert np.array_equal(got[:, 1:5], tlwh), "%s: %s boxes" % (where, which)


def test_nsa_kalman_kernels_with_confidence():
    """b2t_kalman_project / b2t_kalman_update under kalman_format='strongsort' with a confidence: from the float32 mean of a new
    track (FLAG_MEAN_F32: the (1 - conf)-scaled noise is squared in float32) and from a float64 mean, against NSAKalmanFilter."""
    g, lib, fmt = LG.load(), sim(), L.FMT_NSA
    n = len(g["nsa_z0"])
    z0 = g["nsa_z0"].astype(np.float64)
    mean, cov = np.zeros((n, 8)), np.zeros((n, 8, 8))
    L.check(lib, lib.b2t_kalman_initiate(L.F64, fmt, ptr(z0), ptr(mean), ptr(cov), n, None))
    assert np.array_equal(mean, g["nsa_init_mean"].astype(np.float64)) and np.array_equal(cov, g["nsa_init_cov"])
    flags = np.full(n, L.FLAG_MEAN_F32, np.int32)
    for k, (fl, pm_key, ps_key) in enumerate(((flags, "nsa_proj32_mean", "nsa_proj32_cov"), (None, "nsa_proj64_mean", "nsa_proj64_cov"))):
        conf = np.ascontiguousarray(g["nsa_conf%d" % k])
        pm, ps = np.zeros((n, 4)), np.zeros((n, 4, 4))
        L.check(lib, lib.b2t_kalman_project(L.F64, fmt, ptr(mean), ptr(cov), ptr(fl), ptr(conf), ptr(pm), ps.ctypes.data_as(C.c_void_p), n, None))
        if k == 0:      # identical inputs: identical bits
            assert np.array_equal(pm, g[pm_key]) and np.array_equal(ps, g[ps_key])
        np.testing.assert_allclose(pm, g[pm_key], rtol=1e-11, atol=1e-11)
        np.testing.assert_allclose(ps, g[ps_key], rtol=1e-9, atol=1e-11)
        z = np.ascontiguousarray(g["nsa_z%d" % (k + 1)].astype(np.float64))
        conf_u = np.ascontiguousarray(g["nsa_conf%d" % (2 * k)])
        L.check(lib, lib.b2t_kalman_update(L.F64, fmt, ptr(mean), ptr(cov), None, ptr(z), ptr(conf_u), ptr(fl), n, None))
        key = "nsa_upd32" if k == 0 else "nsa_upd64"
        np.testing.assert_allclose(mean, g[key + "_mean"], rtol=1e-11, atol=1e-11)
        np.testing.assert_allclose(cov, g[key + "_cov"], rtol=1e-9, atol=1e-11)
        if k == 0:
            L.check(lib, lib.b2t_kalman_predict(L.F64, fmt, ptr(mean), ptr(cov), None, n, 0, None))
            np.testing.assert_allclose(mean, g["nsa_pred_mean"], rtol=1e-11, atol=1e-11)
            np.testing.assert_allclose(cov, g["nsa_pred_cov"], rtol=1e-9, atol=1e-11)


@pytest.mark.parametrize("name", ["bytetrack_strongsort", "botsort_c01_tb10", "sort_c04_tb8"])
def test_fused_step_f32_lifecycle(name):
    """The float32 build on the lifecycle streams: the reference's ids on every frame, boxes within 1e-4 of the float64 reference."""
    cfg = LG.Config(name)
    frames, warps = cfg.stream()
    trk = SimTracker(cfg.kind, dtype=L.F32, kalman_format=cfg.fmt, conf_thresh=cfg.conf_thresh, track_buffer=cfg.track_buffer,
                     frame_rate=cfg.frame_rate, cap=256, dmax=128)
    for i in range(cfg.n_frames):
        res = trk.step([frames[i]], warps=None if warps is None else warps[i].reshape(1, 6))[0]
        assert res[:, 0].astype(np.int64).tolist() == cfg.out_ids[i].tolist(), "%s frame %d" % (name, i + 1)
        if i in cfg.tlwh_frames:
            np.testing.assert_allclose(res[:, 1:5], cfg.tlwh[("out", i)], rtol=1e-4, atol=2e-2)


@pytest.mark.parametrize("n,m,t", [(1, 1, 0.9), (17, 23, 0.9), (64, 64, 0.5), (150, 120, 0.7)])
def test_lap_solve_f32_on_iou_costs(n, m, t):
    """b2t_lap_solve in float32 on IoU-distance problems (non-integer boxes: a unique optimum): index-exact against the float64
    optimum of the float32-rounded costs."""
    from oracle import iou as oiou, lapjv as olap
    lib = sim()
    rng = np.random.default_rng(n * 7 + m)
    a = rng.uniform(0, 500, (n, 2)); a = np.concatenate([a, a + rng.uniform(8, 90, (n, 2))], 1)
    b = a[rng.integers(0, n, m)] + rng.normal(0, 6, (m, 4))
    c32 = np.ascontiguousarray((1.0 - oiou.ious(a, b)).astype(np.float32))
    x, y = np.full(n, -9, np.int32), np.full(m, -9, np.int32)
    ws = np.zeros(lib.b2t_lap_workspace_bytes(L.F32, n, m, 1) + 512, np.uint8)
    L.check(lib, lib.b2t_lap_solve(L.F32, ptr(c32), n, m, m, t, ptr(x), ptr(y), ptr(ws), ws.size, 1, None))
    _, ex, ey = olap.lapjv(c32.astype(np.float64), True, t)
    assert (ex >= 0).sum() > 0
    assert np.array_equal(x, ex) and np.array_equal(y, ey)
