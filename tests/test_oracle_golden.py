"""not-gpu: the oracle restatement against the committed reference outputs (tests/golden)."""
import os

import numpy as np
import pytest

from oracle import kalman as K, trackers as T, iou as oiou, lapjv as olap
from b200track.synth import make_stream, stream_digest, zero_width_stream

GOLDEN = os.path.join(os.path.dirname(__file__), "golden")


def _load(name):
    return np.load(os.path.join(GOLDEN, name), allow_pickle=False)


@pytest.mark.parametrize("name", ["default", "botsort", "strongsort"])
def test_kalman_matches_reference(name):
    g = _load("kalman_%s.npz" % name)
    fmt = K.FMT_BY_NAME[name]
    z0 = g["z0"]
    n = len(z0)
    m0, c0 = zip(*[K.initiate(fmt, z) for z in z0])
    assert np.array_equal(np.stack(m0), g["init_mean"])
    assert np.array_equal(np.stack([np.asarray(c, np.float64) for c in c0]), g["init_cov"])
    mean, cov = K.multi_predict(fmt, np.stack(m0), np.stack(c0), all_f32=True)
    assert np.array_equal(mean, g["pred32_mean"]) and np.array_equal(cov, g["pred32_cov"])
    for k in range(g["upd_z"].shape[0]):
        zk = g["upd_z"][k]
        for i in range(n):
            pm, ps = K.project(fmt, mean[i], cov[i])
            if name != "strongsort":
                assert np.array_equal(pm, g["proj_mean"][k, i]) and np.array_equal(ps, g["proj_cov"][k, i])
        conf = g["conf%d" % k] if name == "strongsort" else np.zeros(n, np.float32)
        um, uc = zip(*[K.update(fmt, mean[i], cov[i], zk[i], confidence=conf[i]) for i in range(n)])
        assert np.array_equal(np.stack(um), g["upd_mean"][k])
        assert np.array_equal(np.stack(uc), g["upd_cov"][k])
        mean, cov = K.multi_predict(fmt, np.stack(um), np.stack(uc))
        assert np.array_equal(mean, g["pred_mean%d" % k]) and np.array_equal(cov, g["pred_cov%d" % k])
    if name != "strongsort":
        um, uc = zip(*[K.update(fmt, m0[i], c0[i], g["upd_z"][0][i], mean_f32=True) for i in range(n)])
        assert np.array_equal(np.stack(um), g["upd32_mean"]) and np.array_equal(np.stack(uc), g["upd32_cov"])
    if "gate" in g.files and name == "default":
        gate = np.stack([K.gating_distance(fmt, mean[i], cov[i], z0[:8].astype(np.float64)) for i in range(16)])
        np.testing.assert_allclose(gate, g["gate"], rtol=1e-12)


@pytest.mark.parametrize("kind", ["sort", "bytetrack", "botsort"])
@pytest.mark.parametrize("case", ["small", "c3"])
def test_loop_matches_reference(kind, case):
    g = _load("loop_%s.npz" % kind)
    seed, n_obj, n_frames = [int(v) for v in g[case + "_cfg"]]
    frames, warps = make_stream(seed, n_frames, n_obj, warp_sigma=3.0 if kind == "botsort" else 0.0)
    assert stream_digest(frames) == str(g[case + "_digest"]), "synthetic stream generator drifted"
    trk = T.TrackerOracle(kind)
    ids, counts, tl = [], [], {}
    for i, f in enumerate(frames):
        out = trk.update(f, warps[i] if kind == "botsort" else None)
        ids += [o[0] for o in out]
        counts.append(len(out))
        tl[i] = np.array([o[1] for o in out]).reshape(-1, 4)
        assert len(trk.tracked) == g[case + "_ntracked"][i] and len(trk.lost) == g[case + "_nlost"][i]
    assert np.array_equal(np.array(counts), g[case + "_count"])
    assert np.array_equal(np.array(ids), g[case + "_ids"])          # integer ids: bit exact
    got = np.concatenate([tl[int(i)] for i in g[case + "_tlwh_frames"]])
    np.testing.assert_allclose(got, g[case + "_tlwh"], rtol=1e-9, atol=1e-9)


def test_iou_lap_regression():
    g = _load("iou_lap.npz")
    assert np.array_equal(oiou.ious(g["a"], g["b"]), g["iou"])
    adv = oiou.ious(g["adv_a"], g["adv_b"])
    assert np.array_equal(adv, g["adv_iou"])
    # hand-checked "+1" convention values: x2=20 vs x1=21 -> iw = 0 (disjoint);
    # corners sharing pixel (20,20) -> 1 px of overlap between two 11x11 boxes
    assert adv[0, 0] == 0.0
    assert adv[1, 1] == pytest.approx(1.0 / (121 + 121 - 1))
    assert adv[3, 3] == 1.0 and adv[4, 4] == 0.0 and adv[5, 5] == 1.0
    cost = 1.0 - g["iou"]
    for t in (0.9, 0.5, 0.7):
        _, x, y = olap.lapjv(cost, True, t)
        assert np.array_equal(x, g["x_%02d" % int(t * 10)]) and np.array_equal(y, g["y_%02d" % int(t * 10)])


def test_lap_restatement_is_optimal_bruteforce():
    rng = np.random.default_rng(3)
    for _ in range(60):
        n, m = rng.integers(1, 5), rng.integers(1, 5)
        cost = rng.uniform(0, 1, (n, m))
        t = float(rng.choice([0.5, 0.7, 0.9]))
        _, x, y = olap.lapjv(cost, True, t)
        best, bx, uniq = olap.brute_force(cost, t)
        assert olap.objective(cost, x, t) == pytest.approx(best, abs=1e-12)
        if uniq:
            assert np.array_equal(x, bx)
        for i, j in enumerate(x):
            if j >= 0:
                assert y[j] == i and cost[i, j] < t


def test_linear_assignment_empty_sides():
    m, ua, ub = olap.linear_assignment(np.zeros((0, 5)), 0.9)
    assert m.shape == (0, 2) and ua == () and ub == (0, 1, 2, 3, 4)
    m, ua, ub = olap.linear_assignment(np.zeros((3, 0)), 0.9)
    assert m.shape == (0, 2) and ua == (0, 1, 2) and ub == ()


@pytest.mark.parametrize("kind", ["sort", "bytetrack"])
def test_oracle_tracks_zero_width_boxes_like_reference(kind):
    """Boxes flattened to zero width (x2 = x1, height kept) are defined for the xyah Kalman filter -- aspect ratio 0 -- and the
    reference tracks them: the oracle gives the reference's ids on every frame and its boxes on the last (tests/golden/refchecks.npz)."""
    g = _load("refchecks.npz")
    orc = T.TrackerOracle(kind)
    counts = g["flat_%s_count" % kind]
    off = np.concatenate([[0], np.cumsum(counts)])
    for i, f in enumerate(zero_width_stream(61, len(counts), 60)):
        exp = orc.update(f)
        assert [e[0] for e in exp] == g["flat_%s_ids" % kind][off[i]:off[i + 1]].tolist(), "frame %d" % (i + 1)
    np.testing.assert_allclose(np.array([e[1] for e in exp]), g["flat_%s_tlwh_last" % kind], rtol=1e-9, atol=1e-9)
