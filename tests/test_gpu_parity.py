"""-m gpu: the nvcc-built libb200track.so on an H100 against the oracle and the reference goldens.
Everything goes through the C ABI (b200track._lib / engine); nothing here reads the reference tree."""
import os

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

torch = pytest.importorskip("torch")

from b200track import _lib as L                      # noqa: E402
from b200track.synth import make_stream              # noqa: E402
from oracle import kalman as K, iou as oiou, lapjv as olap, trackers as T   # noqa: E402

GOLDEN = os.path.join(os.path.dirname(__file__), "golden")


@pytest.fixture(scope="module")
def ops():
    from b200track.engine import ops as get_ops
    return get_ops()


def _d(ops, a, dt=torch.float64):
    return ops.dev(np.ascontiguousarray(a), dt)


@pytest.mark.parametrize("name", ["default", "botsort", "strongsort"])
def test_kalman_vs_reference_golden(ops, name):
    g = np.load(os.path.join(GOLDEN, "kalman_%s.npz" % name))
    fmt = L.FMT_BY_NAME[name]
    z0 = g["z0"].astype(np.float64); n = len(z0)
    mean, cov = ops.kalman_initiate(L.F64, fmt, _d(ops, z0))
    assert np.array_equal(mean.cpu().numpy(), g["init_mean"].astype(np.float64))
    assert np.array_equal(cov.cpu().numpy(), g["init_cov"])
    m32, c32 = mean.clone(), cov.clone()
    ops.kalman_predict(L.F64, fmt, mean, cov, None, True)
    assert np.array_equal(mean.cpu().numpy(), g["pred32_mean"]) and np.array_equal(cov.cpu().numpy(), g["pred32_cov"])
    for k in range(g["upd_z"].shape[0]):
        pm, ps = ops.kalman_project(L.F64, fmt, mean, cov)
        if name != "strongsort":
            np.testing.assert_allclose(pm.cpu().numpy(), g["proj_mean"][k], rtol=1e-11, atol=1e-11)
            np.testing.assert_allclose(ps.cpu().numpy(), g["proj_cov"][k], rtol=1e-9, atol=1e-11)
        conf = _d(ops, g["conf%d" % k], torch.float32) if name == "strongsort" else None
        ops.kalman_update(L.F64, fmt, mean, cov, _d(ops, g["upd_z"][k].astype(np.float64)), None, conf, None)
        np.testing.assert_allclose(mean.cpu().numpy(), g["upd_mean"][k], rtol=1e-11, atol=1e-11)   # tolerance: north_star 1e-4
        np.testing.assert_allclose(cov.cpu().numpy(), g["upd_cov"][k], rtol=1e-9, atol=1e-11)
        ops.kalman_predict(L.F64, fmt, mean, cov, None, False)
        np.testing.assert_allclose(mean.cpu().numpy(), g["pred_mean%d" % k], rtol=1e-11, atol=1e-11)
        np.testing.assert_allclose(cov.cpu().numpy(), g["pred_cov%d" % k], rtol=1e-9, atol=1e-11)
    if name != "strongsort":
        flags = _d(ops, np.full(n, L.FLAG_MEAN_F32, np.int32), torch.int32)
        ops.kalman_update(L.F64, fmt, m32, c32, _d(ops, g["upd_z"][0].astype(np.float64)), None, None, flags)
        np.testing.assert_allclose(m32.cpu().numpy(), g["upd32_mean"], rtol=1e-11, atol=1e-11)
        np.testing.assert_allclose(c32.cpu().numpy(), g["upd32_cov"], rtol=1e-9, atol=1e-11)
    if "gate" in g.files and name == "default":
        for i in range(4):
            got = ops.kalman_gating(L.F64, fmt, mean[i], cov[i], _d(ops, z0[:8])).cpu().numpy()
            np.testing.assert_allclose(got, g["gate"][i], rtol=1e-9)


def test_kalman_f32_mode_meets_1e4(ops):
    g = np.load(os.path.join(GOLDEN, "kalman_default.npz"))
    z0 = g["z0"].astype(np.float32)
    mean, cov = ops.kalman_initiate(L.F32, 0, _d(ops, z0, torch.float32))
    ops.kalman_predict(L.F32, 0, mean, cov, None, True)
    for k in range(3):
        ops.kalman_update(L.F32, 0, mean, cov, _d(ops, g["upd_z"][k], torch.float32))
        np.testing.assert_allclose(mean.cpu().numpy()[:, :4], g["upd_mean"][k][:, :4], rtol=1e-4, atol=1e-4)
        ops.kalman_predict(L.F32, 0, mean, cov, None, False)


def test_gmc_vs_oracle(ops):
    rng = np.random.default_rng(0)
    n = 1000
    mean = rng.normal(0, 50, (n, 8)); a = rng.normal(0, 1, (n, 8, 8)); cov = a @ a.transpose(0, 2, 1)
    warp = np.array([[0.99, -0.02, 3.5], [0.02, 1.01, -1.25]])
    em, ec = K.gmc_apply(mean, cov, warp)
    dm, dc = _d(ops, mean), _d(ops, cov)
    ops.gmc_apply(L.F64, dm, dc, warp)
    np.testing.assert_allclose(dm.cpu().numpy(), em, rtol=1e-13, atol=1e-12)
    np.testing.assert_allclose(dc.cpu().numpy(), ec, rtol=1e-12, atol=1e-10)


def _boxes(rng, k, span=1200):
    p = np.round(rng.uniform(0, span, (k, 2)))
    return np.concatenate([p, p + np.round(rng.uniform(4, 120, (k, 2)))], 1)


@pytest.mark.parametrize("n,m", [(1, 1), (48, 40), (300, 257), (1024, 999), (2048, 2048)])
def test_iou_bit_exact(ops, n, m):
    rng = np.random.default_rng(n * 1000 + m)
    a, b = _boxes(rng, n) + rng.choice([0, 0.5], (n, 1)), _boxes(rng, m)
    cost = ops.iou_cost(L.F64, _d(ops, a), _d(ops, b)).cpu().numpy()
    assert np.array_equal(cost, 1.0 - oiou.ious(a, b))                # integer / byte-exact contract: fp64 bit equality
    c32 = ops.iou_cost(L.F32, _d(ops, a, torch.float32), _d(ops, b, torch.float32)).cpu().numpy()
    np.testing.assert_allclose(c32, cost, atol=2e-6)                  # SURVEY section 4: IoU abs 1e-6 class


def test_iou_batched(ops):
    rng = np.random.default_rng(9)
    a = np.stack([_boxes(rng, 64) for _ in range(5)]); b = np.stack([_boxes(rng, 50) for _ in range(5)])
    cost = ops.iou_cost(L.F64, _d(ops, a), _d(ops, b)).cpu().numpy()
    for i in range(5):
        assert np.array_equal(cost[i], 1.0 - oiou.ious(a[i], b[i]))


def _iou_problem(rng, n, m, span):
    a = _boxes(rng, n, span)
    b = a[rng.integers(0, n, m)] + np.round(rng.normal(0, 4, (m, 4)))
    return 1.0 - oiou.ious(a, b)


@pytest.mark.parametrize("n,m,t,span", [(60, 47, 0.9, 500), (300, 280, 0.9, 1200), (300, 280, 0.5, 1200), (257, 1024, 0.7, 2500),
                                         (1024, 1024, 0.9, 2500), (2048, 2048, 0.9, 4000), (2048, 2048, 0.5, 4000)])
def test_lap_vs_oracle(ops, n, m, t, span):
    rng = np.random.default_rng(n + 7 * m)
    cost = _iou_problem(rng, n, m, span)
    x, y = ops.lap_solve(L.F64, _d(ops, cost), t)
    x, y = x.cpu().numpy(), y.cpu().numpy()
    _, ex, ey = olap.lapjv(cost, True, t)
    assert olap.objective(cost, x, t) == pytest.approx(olap.objective(cost, ex, t), abs=1e-8)
    assert np.array_equal(x, ex) and np.array_equal(y, ey)           # indices: bit-exact contract
    for i, j in enumerate(x):                                        # structural properties at full size
        if j >= 0:
            assert y[j] == i and cost[i, j] < t


def test_lap_dense_random_and_batched(ops):
    rng = np.random.default_rng(4)
    cost = rng.uniform(0, 1, (6, 90, 70))
    x, y = ops.lap_solve(L.F64, _d(ops, cost), 2.0)                  # every entry eligible: one big component
    for i in range(6):
        _, ex, ey = olap.lapjv(cost[i], True, 2.0)
        assert olap.objective(cost[i], x[i].cpu().numpy(), 2.0) == pytest.approx(olap.objective(cost[i], ex, 2.0), abs=1e-9)
        assert np.array_equal(x[i].cpu().numpy(), ex)


def test_lap_empty_and_all_gated(ops):
    cost = np.full((30, 20), 0.95)
    x, y = ops.lap_solve(L.F64, _d(ops, cost), 0.9)
    assert (x.cpu().numpy() == -1).all() and (y.cpu().numpy() == -1).all()


def _run_engine(kind, frames, warps, dtype="f64", cap=512, dmax=512):
    from b200track.engine import TrackEngine
    eng = TrackEngine(kind, n_seq=1, dtype=dtype, cap=cap, dmax=dmax)
    res = []
    for i, f in enumerate(frames):
        res.append(eng.step([f], warps=warps[i].reshape(1, 6) if kind == "botsort" else None)[0].copy())
    return res


@pytest.mark.parametrize("kind", ["sort", "bytetrack", "botsort"])
@pytest.mark.parametrize("case", ["small", "c3"])
def test_fused_step_matches_reference_golden(kind, case):
    g = np.load(os.path.join(GOLDEN, "loop_%s.npz" % kind))
    seed, n_obj, n_frames = [int(v) for v in g[case + "_cfg"]]
    frames, warps = make_stream(seed, n_frames, n_obj, warp_sigma=3.0 if kind == "botsort" else 0.0)
    res = _run_engine(kind, frames, warps)
    counts = g[case + "_count"]
    off = np.concatenate([[0], np.cumsum(counts)])
    keep = {int(f): i for i, f in enumerate(g[case + "_tlwh_frames"])}
    tl_off = np.concatenate([[0], np.cumsum(counts[g[case + "_tlwh_frames"]])])
    for i in range(n_frames):
        assert np.array_equal(res[i][:, 0].astype(np.int64), g[case + "_ids"][off[i]:off[i + 1]]), "ids differ at frame %d" % (i + 1)
        assert np.array_equal(res[i][:, 5].astype(np.float32), g[case + "_cls"][off[i]:off[i + 1]])
        if i in keep:
            k = keep[i]
            np.testing.assert_allclose(res[i][:, 1:5], g[case + "_tlwh"][tl_off[k]:tl_off[k + 1]], rtol=1e-9, atol=1e-9)


@pytest.mark.parametrize("kind", ["bytetrack", "botsort", "sort"])
def test_fused_step_vs_oracle_multi_sequence(kind):
    """4 sequences of ~300 detections advanced together (BASELINE config C3 shape), fresh seeds."""
    from b200track.engine import TrackEngine
    S, F = 4, 90
    streams = [make_stream(500 + s, F, 300, warp_sigma=3.0 if kind == "botsort" else 0.0) for s in range(S)]
    eng = TrackEngine(kind, n_seq=S, cap=1024, dmax=512)
    orcs = [T.TrackerOracle(kind) for _ in range(S)]
    for i in range(F):
        warps = np.stack([streams[s][1][i].reshape(6) for s in range(S)]) if kind == "botsort" else None
        got = eng.step([streams[s][0][i] for s in range(S)], warps=warps)
        for s in range(S):
            exp = orcs[s].update(streams[s][0][i], streams[s][1][i] if kind == "botsort" else None)
            assert [int(v) for v in got[s][:, 0]] == [e[0] for e in exp], "seq %d frame %d" % (s, i + 1)
            if exp:
                np.testing.assert_allclose(got[s][:, 1:5], np.array([e[1] for e in exp]), rtol=1e-9, atol=1e-9)
            assert eng.np_stat[s, L.STAT_NTRACKED] == len(orcs[s].tracked) and eng.np_stat[s, L.STAT_NLOST] == len(orcs[s].lost)


@pytest.mark.parametrize("kind", ["bytetrack", "botsort", "sort"])
def test_fused_step_ignores_boxes_without_area(kind):
    """Boxes the reference cannot track (zero height, non-finite, and zero width under the xywh filter; scale_coords' clip + round
    flattens boxes off the image edge, and the benchmark's noise detector makes many per frame) take no part: 4 sequences with such
    boxes inserted give the tracks of the clean streams (oracle), and every output is finite."""
    from b200track.engine import TrackEngine
    from b200track.synth import with_flat_boxes
    S, F = 4, 60
    streams = [make_stream(800 + s, F, 300, warp_sigma=3.0 if kind == "botsort" else 0.0) for s in range(S)]
    rng = np.random.default_rng(9)
    dirty = [[with_flat_boxes(f, rng, xywh=kind == "botsort") for f in streams[s][0]] for s in range(S)]
    eng = TrackEngine(kind, n_seq=S, cap=1024, dmax=512)
    orcs = [T.TrackerOracle(kind) for _ in range(S)]
    for i in range(F):
        warps = np.stack([streams[s][1][i].reshape(6) for s in range(S)]) if kind == "botsort" else None
        got = eng.step([dirty[s][i] for s in range(S)], warps=warps)
        for s in range(S):
            exp = orcs[s].update(streams[s][0][i], streams[s][1][i] if kind == "botsort" else None)
            assert np.isfinite(got[s]).all(), "seq %d frame %d" % (s, i + 1)
            assert [int(v) for v in got[s][:, 0]] == [e[0] for e in exp], "seq %d frame %d" % (s, i + 1)
            if exp:
                np.testing.assert_allclose(got[s][:, 1:5], np.array([e[1] for e in exp]), rtol=1e-9, atol=1e-9)


@pytest.mark.parametrize("kind", ["sort", "bytetrack"])
def test_fused_step_tracks_zero_width_boxes_like_reference(kind):
    """Zero-width, positive-height boxes are defined for the xyah filter and the reference tracks them: the fused step gives the
    reference's ids (tests/golden/refchecks.npz) on every frame and its boxes on the last."""
    from b200track.engine import TrackEngine
    from b200track.synth import zero_width_stream
    g = np.load(os.path.join(os.path.dirname(__file__), "golden", "refchecks.npz"))
    counts = g["flat_%s_count" % kind]
    off = np.concatenate([[0], np.cumsum(counts)])
    eng = TrackEngine(kind, n_seq=1, cap=256, dmax=128)
    for i, f in enumerate(zero_width_stream(61, len(counts), 60)):
        got = eng.step([f])[0]
        assert got[:, 0].astype(np.int64).tolist() == g["flat_%s_ids" % kind][off[i]:off[i + 1]].tolist(), "frame %d" % (i + 1)
    np.testing.assert_allclose(got[:, 1:5], g["flat_%s_tlwh_last" % kind], rtol=1e-9, atol=1e-9)


@pytest.mark.parametrize("kind", ["bytetrack", "botsort"])
def test_fused_step_crowded_scene_spills_edges(kind):
    """300 objects inside a 300 x 300 px area: ~9 000 sub-threshold pairs per association, far more than the shared-memory edge mirror
    holds -- rows live in the mirror, in the second window (the idle box arrays) and in the global workspace, and the augmenting searches
    run long.  Ids and boxes equal the oracle's frame by frame (the simulator runs the same stream in tests/test_hostsim_logic.py)."""
    from b200track.engine import TrackEngine
    frames, warps = make_stream(77, 20, 300, img=700, warp_sigma=2.0 if kind == "botsort" else 0.0)
    eng = TrackEngine(kind, n_seq=1, cap=1024, dmax=512)
    orc = T.TrackerOracle(kind)
    for i, f in enumerate(frames):
        got = eng.step([f], warps=warps[i].reshape(1, 6) if kind == "botsort" else None)[0]
        exp = orc.update(f, warps[i] if kind == "botsort" else None)
        assert eng.np_stat[0, L.STAT_ERR] == 0
        assert [int(v) for v in got[:, 0]] == [e[0] for e in exp], "frame %d" % (i + 1)
        if exp:
            np.testing.assert_allclose(got[:, 1:5], np.array([e[1] for e in exp]), rtol=1e-9, atol=1e-9)
    assert int(eng.np_stat[0, 15]) > 8000


def test_fused_step_f32_mode():
    """All-fp32 arithmetic: boxes within the north_star tolerance (1e-4 rel) of the fp64 reference
    while the id sequence is identical on this tie-free stream."""
    g = np.load(os.path.join(GOLDEN, "loop_bytetrack.npz"))
    seed, n_obj, n_frames = [int(v) for v in g["small_cfg"]]
    frames, warps = make_stream(seed, n_frames, n_obj)
    res = _run_engine("bytetrack", frames, warps, dtype="f32")
    counts = g["small_count"]; off = np.concatenate([[0], np.cumsum(counts)])
    keep = {int(f): i for i, f in enumerate(g["small_tlwh_frames"])}
    tl_off = np.concatenate([[0], np.cumsum(counts[g["small_tlwh_frames"]])])
    for i in range(n_frames):
        assert np.array_equal(res[i][:, 0].astype(np.int64), g["small_ids"][off[i]:off[i + 1]])
        if i in keep:
            k = keep[i]
            np.testing.assert_allclose(res[i][:, 1:5], g["small_tlwh"][tl_off[k]:tl_off[k + 1]], rtol=1e-4, atol=2e-2)


def test_update_without_detection_and_slot_readback():
    from b200track.engine import TrackEngine
    frames, _ = make_stream(31, 6, 25)
    eng = TrackEngine("bytetrack", cap=128, dmax=128)
    orc = T.TrackerOracle("bytetrack")
    for i in range(4):
        eng.step([frames[i]]); orc.update(frames[i])
    r = eng.step(None, predict_only=True)[0]
    e = orc.update_without_detection()
    assert [int(v) for v in r[:, 0]] == [x[0] for x in e]
    np.testing.assert_allclose(r[:, 1:5], np.array([x[1] for x in e]), rtol=1e-12, atol=1e-9)
    slot = int(r[0, 7])
    mean, cov = eng.read_slot(0, slot)
    tid = int(r[0, 0])
    ref = [t for t in orc.trk.values() if t.tid == tid][0]
    np.testing.assert_allclose(mean, ref.mean, rtol=1e-11, atol=1e-11)
    np.testing.assert_allclose(cov, ref.cov, rtol=1e-9, atol=1e-11)


def test_capacity_errors_are_loud():
    from b200track.engine import TrackEngine
    frames, _ = make_stream(3, 3, 120)
    eng = TrackEngine("bytetrack", cap=64, dmax=256)        # 64 slots cannot hold ~110 births
    with pytest.raises(L.B2TError):
        for f in frames:
            eng.step([f])


def test_dropin_modules_end_to_end():
    """The reference-facing surface: bare-name modules, ByteTrack(opts).update(dets, img) -> STrack list."""
    import sys
    tdir = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "yolov7-tracker_b200", "tracker")
    sys.path.insert(0, tdir)
    try:
        import basetrack, bytetrack, botsort, matching, kalman_filter
    finally:
        sys.path.remove(tdir)

    class Opts:
        conf_thresh = 0.2; track_buffer = 30; kalman_format = "default"; img_size = 1280; iou_thresh = 0.5
        reid_model_path = ""; dhn_path = ""; b2t_cap = 256; b2t_dmax = 256

    g = np.load(os.path.join(GOLDEN, "loop_bytetrack.npz"))
    seed, n_obj, n_frames = [int(v) for v in g["small_cfg"]]
    frames, _ = make_stream(seed, n_frames, n_obj)
    basetrack.BaseTrack._count = 0
    trk = bytetrack.ByteTrack(Opts(), frame_rate=30)
    off = np.concatenate([[0], np.cumsum(g["small_count"])])
    img = torch.zeros((4, 4, 3), dtype=torch.uint8)
    for i in range(40):
        cur = trk.update(torch.from_numpy(frames[i]).cuda(), img)       # CUDA tensor input, as track.py:151 passes it
        assert [t.track_id for t in cur] == list(g["small_ids"][off[i]:off[i + 1]])
        assert all(t.tlwh.shape == (4,) for t in cur)
    assert cur[0].mean.shape == (8,) and cur[0].cov.shape == (8, 8)      # lazy device read-back
    assert basetrack.BaseTrack._count == g["small_ids"][:off[40]].max()
    # op-level API: same call shapes as the reference modules
    kf = kalman_filter.KalmanFilter()
    m, c = kf.initiate(np.array([100., 200., 0.5, 80.], np.float32))
    em, ec = K.initiate(0, np.array([100., 200., 0.5, 80.], np.float32))
    assert m.dtype == np.float32 and np.array_equal(m, em) and np.array_equal(c, ec)
    m1, c1 = kf.predict(m, c)
    e1, f1 = K.multi_predict(0, em[None], ec[None], all_f32=True)
    assert np.array_equal(m1, e1[0]) and np.array_equal(c1, f1[0])
    m2, c2 = kf.update(m1, c1, np.array([101., 201., 0.5, 81.], np.float32))
    e2, f2 = K.update(0, e1[0], f1[0], np.array([101., 201., 0.5, 81.], np.float32))
    np.testing.assert_allclose(m2, e2, rtol=1e-11); np.testing.assert_allclose(c2, f2, rtol=1e-8, atol=1e-12)
    rng = np.random.default_rng(1)
    a, b = _boxes(rng, 30), _boxes(rng, 25)
    cost = matching.iou_distance([r for r in a], [r for r in b])
    assert np.array_equal(cost, 1 - oiou.ious(a, b))
    mt, ua, ub = matching.linear_assignment(cost, 0.9)
    em_, eua, eub = olap.linear_assignment(cost, 0.9)
    assert np.array_equal(np.asarray(mt).reshape(-1, 2), np.asarray(em_).reshape(-1, 2)) and np.array_equal(ua, eua) and np.array_equal(ub, eub)
    mt, ua, ub = matching.linear_assignment(np.zeros((0, 3)), 0.9)
    assert mt.shape == (0, 2) and ua == () and ub == (0, 1, 2)


# ------------------------------------------------------------------------------------------ round 2 additions
def _valid_matching(cost, x, y, t):
    n, m = cost.shape
    for i, j in enumerate(x):
        if j >= 0:
            assert 0 <= j < m and y[j] == i and cost[i, j] < t
    for j, i in enumerate(y):
        if i >= 0:
            assert x[i] == j
    assert len({j for j in x if j >= 0}) == int((x >= 0).sum())


def test_lap_ties_and_duplicate_boxes(ops):
    """Equal-cost optima: duplicated detections / duplicated tracks make several assignments optimal, so the INDEX contract
    cannot hold (any exact solver may pick any optimum -- SURVEY 7.2 #2); what must hold is a valid matching with the optimal
    objective of sum(c - t), on the device as in the oracle.  Also an all-equal matrix and a matrix of exact zeros."""
    rng = np.random.default_rng(77)
    a = _boxes(rng, 120, 900)
    a[60:] = a[:60]                                                   # every track box twice
    b = np.concatenate([a[:40], a[:40], _boxes(rng, 30, 900)])        # detections: 40 boxes twice + 30 strangers
    cost = 1.0 - oiou.ious(a, b)
    for t in (0.9, 0.5):
        x, y = ops.lap_solve(L.F64, _d(ops, cost), t)
        x, y = x.cpu().numpy(), y.cpu().numpy()
        _valid_matching(cost, x, y, t)
        _, ex, _ = olap.lapjv(cost, True, t)
        assert olap.objective(cost, x, t) == pytest.approx(olap.objective(cost, ex, t), abs=1e-9)
        assert int((x >= 0).sum()) == int((ex >= 0).sum())            # same cardinality: every zero-cost duplicate pair is worth matching
    flat = np.full((16, 12), 0.25)
    x, y = ops.lap_solve(L.F64, _d(ops, flat), 0.9)
    x, y = x.cpu().numpy(), y.cpu().numpy()
    _valid_matching(flat, x, y, 0.9)
    assert int((x >= 0).sum()) == 12                                  # all-equal costs: any perfect matching of the smaller side
    zeros = np.zeros((9, 9))
    x, y = ops.lap_solve(L.F64, _d(ops, zeros), 0.5)
    assert int((x.cpu().numpy() >= 0).sum()) == 9


def test_iou_lap_property_sweep(ops):
    """hypothesis: N, M in [0, 2048] (empty sides included), random thresholds: IoU bit-equal to the oracle, LAP a valid matching
    with the oracle's objective (indices equal whenever the oracle says the optimum is unique on small problems)."""
    hyp = pytest.importorskip("hypothesis")
    from hypothesis import given, settings, strategies as st, HealthCheck

    @settings(max_examples=25, deadline=None, suppress_health_check=list(HealthCheck), derandomize=True)
    @given(n=st.one_of(st.integers(0, 40), st.integers(0, 2048)), m=st.one_of(st.integers(0, 40), st.integers(0, 2048)),
           t=st.sampled_from([0.5, 0.7, 0.9]), seed=st.integers(0, 2 ** 16))
    def run(n, m, t, seed):
        rng = np.random.default_rng(seed)
        a, b = _boxes(rng, n, 1500), _boxes(rng, m, 1500)
        if n and m:
            k = min(n, m)
            b[:k] = a[rng.permutation(n)[:k]] + np.round(rng.normal(0, 3, (k, 4)))     # real overlaps
        cost = ops.iou_cost(L.F64, _d(ops, a.reshape(n, 4)), _d(ops, b.reshape(m, 4))).cpu().numpy() if n and m else np.zeros((n, m))
        if n and m:
            assert np.array_equal(cost, 1.0 - oiou.ious(a, b))
        if n == 0 or m == 0:
            return                                                    # matching.linear_assignment short-circuits on the host (matching.py:31-32)
        x, y = ops.lap_solve(L.F64, _d(ops, cost), t)
        x, y = x.cpu().numpy(), y.cpu().numpy()
        _valid_matching(cost, x, y, t)
        _, ex, ey = olap.lapjv(cost, True, t)
        assert olap.objective(cost, x, t) == pytest.approx(olap.objective(cost, ex, t), abs=1e-8)
    run()


def test_botsort_c4_size_vs_oracle():
    """BASELINE config C4 shape: BoT-SORT (Kalman xywh + per-frame camera warp + IoU), 500 objects per frame, the sequences of
    one GPU advanced together, every frame against the oracle: ids exact, boxes 1e-9, pool sizes equal (q3 / q4 duplicates
    included: the id counter runs well past the object count)."""
    from b200track.engine import TrackEngine
    S, F = 2, 45
    streams = [make_stream(4000 + s, F, 500, warp_sigma=3.0) for s in range(S)]
    eng = TrackEngine("botsort", n_seq=S, cap=1152, dmax=576)          # one CTA per sequence: its working set must fit 227 KB of shared memory
    orcs = [T.TrackerOracle("botsort") for _ in range(S)]
    for i in range(F):
        warps = np.stack([streams[s][1][i].reshape(6) for s in range(S)])
        got = eng.step([streams[s][0][i] for s in range(S)], warps=warps)
        for s in range(S):
            exp = orcs[s].update(streams[s][0][i], streams[s][1][i])
            assert [int(v) for v in got[s][:, 0]] == [e[0] for e in exp], "seq %d frame %d" % (s, i + 1)
            if exp:
                np.testing.assert_allclose(got[s][:, 1:5], np.array([e[1] for e in exp]), rtol=1e-9, atol=1e-9)
            assert eng.np_stat[s, L.STAT_NTRACKED] == len(orcs[s].tracked) and eng.np_stat[s, L.STAT_NLOST] == len(orcs[s].lost)
    assert int(eng.np_stat[0, L.STAT_NEXT_ID]) > 500 and int(eng.np_stat[0, L.STAT_ERR]) == 0


def test_output_row_overflow_sets_error_bit():
    """More confirmed tracks than output rows: the kernel drops rows AND raises ERR_OUT (it used to clamp silently)."""
    from b200track.engine import TrackEngine
    frames, _ = make_stream(5, 3, 60)
    eng = TrackEngine("bytetrack", n_seq=1, cap=256, dmax=128)
    eng.set_out_rows(16)
    with pytest.raises(L.B2TError):
        for f in frames:
            eng.step([f])


def test_embedding_distance_on_tensor_cores_matches_float64():
    """matching.embedding_distance / cal_cosine_distance (tracker/matching.py:84-103, 165-178): the N x 512 x M cosine GEMM runs on the
    wgmma conv kernel with split-fp16 operands and must reproduce NumPy's float64 result to ~1e-6 (the appearance costs feed the same
    thresholded assignment as the IoU costs)."""
    import sys
    tdir = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "yolov7-tracker_b200", "tracker")
    sys.path.insert(0, tdir)
    try:
        import matching
    finally:
        sys.path.remove(tdir)
    rng = np.random.default_rng(12)

    class T_:
        def __init__(self, f):
            self.features = [f]
    for n, m, d in ((37, 51, 512), (300, 280, 512), (5, 700, 512), (130, 3, 128)):
        a, b = rng.normal(0, 1, (n, d)), rng.normal(0, 1, (m, d)) * rng.uniform(0.1, 10, (m, 1))
        b[: min(n, m)] = a[: min(n, m)] + rng.normal(0, 0.05, (min(n, m), d))                # near-duplicates: similarities close to 1
        ref = (a / np.linalg.norm(a, axis=1, keepdims=True)) @ (b / np.linalg.norm(b, axis=1, keepdims=True)).T
        got = matching.cal_cosine_distance(a, b)
        assert got.shape == ref.shape and np.abs(got - ref).max() < 5e-6, (n, m, d, np.abs(got - ref).max())
        cost = matching.embedding_distance([T_(r) for r in a], [T_(r) for r in b])
        assert np.abs(cost - (1.0 - ref)).max() < 5e-6
    assert matching.embedding_distance([], [T_(b[0])]).shape == (0, 1)
