"""not-gpu: kernel LOGIC of csrc/b2t_*.cuh, executed by the fiber simulator (tests/hostsim), against
the oracle and the committed reference goldens.  This tier exists because the CPU test machine
has no GPU; it does not replace the `-m gpu` parity tests, which run the nvcc build on an H100."""
import ctypes as C
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.join(os.path.dirname(__file__), "hostsim"))
import simlib  # noqa: E402
from simlib import ptr, sim, SimTracker  # noqa: E402
from b200track import _lib as L  # noqa: E402
from b200track.synth import make_stream, with_flat_boxes, zero_width_stream  # noqa: E402
from oracle import kalman as K, iou as oiou, lapjv as olap, trackers as T  # noqa: E402

GOLDEN = os.path.join(os.path.dirname(__file__), "golden")


@pytest.mark.parametrize("name", ["default", "botsort", "strongsort"])
def test_kalman_kernels_vs_reference_golden(name):
    g = np.load(os.path.join(GOLDEN, "kalman_%s.npz" % name))
    lib, fmt = sim(), L.FMT_BY_NAME[name]
    z0 = g["z0"].astype(np.float64)
    n = len(z0)
    mean = np.zeros((n, 8)); cov = np.zeros((n, 8, 8))
    L.check(lib, lib.b2t_kalman_initiate(L.F64, fmt, ptr(z0), ptr(mean), ptr(cov), n, None))
    assert np.array_equal(mean, g["init_mean"].astype(np.float64))
    assert np.array_equal(cov, g["init_cov"])
    m32, c32 = mean.copy(), cov.copy()
    L.check(lib, lib.b2t_kalman_predict(L.F64, fmt, ptr(mean), ptr(cov), None, n, 1, None))
    assert np.array_equal(mean, g["pred32_mean"]) and np.array_equal(cov, g["pred32_cov"])
    for k in range(g["upd_z"].shape[0]):
        zk = g["upd_z"][k].astype(np.float64)
        pm = np.zeros((n, 4)); ps = np.zeros((n, 4, 4))
        L.check(lib, lib.b2t_kalman_project(L.F64, fmt, ptr(mean), ptr(cov), None, None, ptr(pm), ptr(ps), n, None))
        if name != "strongsort":
            if k == 0:      # identical inputs -> identical bits; later rounds carry ulp-level history
                assert np.array_equal(pm, g["proj_mean"][k]) and np.array_equal(ps, g["proj_cov"][k])
            np.testing.assert_allclose(pm, g["proj_mean"][k], rtol=1e-11, atol=1e-11)
            np.testing.assert_allclose(ps, g["proj_cov"][k], rtol=1e-9, atol=1e-11)
        conf = np.ascontiguousarray(g["conf%d" % k]) if name == "strongsort" else None
        L.check(lib, lib.b2t_kalman_update(L.F64, fmt, ptr(mean), ptr(cov), None, ptr(zk), ptr(conf), None, n, None))
        np.testing.assert_allclose(mean, g["upd_mean"][k], rtol=1e-11, atol=1e-11)
        np.testing.assert_allclose(cov, g["upd_cov"][k], rtol=1e-9, atol=1e-11)
        L.check(lib, lib.b2t_kalman_predict(L.F64, fmt, ptr(mean), ptr(cov), None, n, 0, None))
        np.testing.assert_allclose(mean, g["pred_mean%d" % k], rtol=1e-11, atol=1e-11)
        np.testing.assert_allclose(cov, g["pred_cov%d" % k], rtol=1e-9, atol=1e-11)
    if name != "strongsort":
        flags = np.full(n, L.FLAG_MEAN_F32, np.int32)
        z = g["upd_z"][0].astype(np.float64)
        L.check(lib, lib.b2t_kalman_update(L.F64, fmt, ptr(m32), ptr(c32), None, ptr(z), None, ptr(flags), n, None))
        np.testing.assert_allclose(m32, g["upd32_mean"], rtol=1e-11, atol=1e-11)
        np.testing.assert_allclose(c32, g["upd32_cov"], rtol=1e-9, atol=1e-11)


def test_kalman_f32_mode_within_tolerance():
    g = np.load(os.path.join(GOLDEN, "kalman_default.npz"))
    lib = sim()
    z0 = g["z0"].astype(np.float32); n = len(z0)
    mean = np.zeros((n, 8), np.float32); cov = np.zeros((n, 8, 8), np.float32)
    L.check(lib, lib.b2t_kalman_initiate(L.F32, 0, ptr(z0), ptr(mean), ptr(cov), n, None))
    L.check(lib, lib.b2t_kalman_predict(L.F32, 0, ptr(mean), ptr(cov), None, n, 1, None))
    zk = np.ascontiguousarray(g["upd_z"][0].astype(np.float32))
    L.check(lib, lib.b2t_kalman_update(L.F32, 0, ptr(mean), ptr(cov), None, ptr(zk), None, None, n, None))
    np.testing.assert_allclose(mean[:, :4], g["upd_mean"][0][:, :4], rtol=1e-4, atol=1e-4)   # north_star tolerance


def test_gmc_kernel_vs_oracle():
    rng = np.random.default_rng(0)
    n = 37
    mean = rng.normal(0, 50, (n, 8)); a = rng.normal(0, 1, (n, 8, 8)); cov = a @ a.transpose(0, 2, 1)
    warp = np.array([[0.99, -0.02, 3.5], [0.02, 1.01, -1.25]])
    em, ec = K.gmc_apply(mean, cov, warp)
    w6 = (C.c_double * 6)(*warp.reshape(-1))
    L.check(sim(), sim().b2t_gmc_apply(L.F64, ptr(mean), ptr(cov), n, w6, None))
    np.testing.assert_allclose(mean, em, rtol=1e-13, atol=1e-12)
    np.testing.assert_allclose(cov, ec, rtol=1e-12, atol=1e-10)


@pytest.mark.parametrize("n,m", [(0, 5), (7, 0), (1, 1), (48, 40), (130, 257)])
def test_iou_kernel_bit_exact(n, m):
    rng = np.random.default_rng(n * 1000 + m)
    def boxes(k):
        p = np.round(rng.uniform(0, 300, (k, 2)))
        return np.concatenate([p, p + np.round(rng.uniform(0, 90, (k, 2)))], 1) + rng.choice([0, 0.5], (k, 1))
    a, b = boxes(n), boxes(m)
    cost = np.full((n, max(m, 1)), -7.0)
    L.check(sim(), sim().b2t_iou_cost(L.F64, ptr(a), n, ptr(b), m, ptr(cost), max(m, 1), 1, 1, None))
    if n and m:
        assert np.array_equal(cost[:, :m], 1.0 - oiou.ious(a, b))     # bit exact


def _lap(cost, thresh, dtype=L.F64):
    lib = sim()
    n, m = cost.shape
    c = np.ascontiguousarray(cost, simlib.npdt(dtype))
    x = np.full(n, -9, np.int32); y = np.full(m, -9, np.int32)
    ws = np.zeros(lib.b2t_lap_workspace_bytes(dtype, n, m, 1) + 512, np.uint8)
    L.check(lib, lib.b2t_lap_solve(dtype, ptr(c), n, m, max(m, 1), thresh, ptr(x), ptr(y), ptr(ws), ws.size, 1, None))
    return x, y


def test_lap_kernel_small_bruteforce():
    rng = np.random.default_rng(5)
    for _ in range(40):
        n, m = int(rng.integers(1, 5)), int(rng.integers(1, 5))
        cost = rng.uniform(0, 1, (n, m))
        t = float(rng.choice([0.5, 0.7, 0.9]))
        x, y = _lap(cost, t)
        best, bx, uniq = olap.brute_force(cost, t)
        assert olap.objective(cost, x, t) == pytest.approx(best, abs=1e-12)
        assert uniq and np.array_equal(x, bx)


@pytest.mark.parametrize("n,m,t", [(0, 4, 0.9), (5, 0, 0.9), (60, 47, 0.9), (60, 47, 0.5), (200, 230, 0.7), (33, 64, 2.0)])
def test_lap_kernel_vs_oracle(n, m, t):
    rng = np.random.default_rng(n + 7 * m)
    if n and m:
        a = np.round(rng.uniform(0, 500, (n, 2))); a = np.concatenate([a, a + np.round(rng.uniform(8, 90, (n, 2)))], 1)
        src = a[rng.integers(0, n, m)]
        b = src + np.round(rng.normal(0, 4, (m, 4)))
        cost = 1.0 - oiou.ious(a, b) if t < 1.5 else rng.uniform(0, 1, (n, m))    # t=2.0: dense, everything eligible
    else:
        cost = np.zeros((n, m))
    x, y = _lap(cost, t)
    if n == 0 or m == 0:
        assert (x == -1).all() and (y == -1).all()
        return
    _, ex, ey = olap.lapjv(cost, True, t)
    assert olap.objective(cost, x, t) == pytest.approx(olap.objective(cost, ex, t), abs=1e-9)
    assert np.array_equal(x, ex) and np.array_equal(y, ey)


def _run_loop(kind, frames, warps, dtype=L.F64, cap=512, dmax=512):
    trk = SimTracker(kind, dtype=dtype, cap=cap, dmax=dmax)
    res = []
    for i, f in enumerate(frames):
        w = warps[i].reshape(1, 6) if kind == "botsort" else None
        res.append(trk.step([f], warps=w)[0])
    return res, trk


@pytest.mark.parametrize("kind", ["sort", "bytetrack", "botsort"])
@pytest.mark.parametrize("case", ["small", "c3"])
def test_fused_step_matches_reference_golden(kind, case):
    g = np.load(os.path.join(GOLDEN, "loop_%s.npz" % kind))
    seed, n_obj, n_frames = [int(v) for v in g[case + "_cfg"]]
    if case == "c3":
        n_frames = 24          # the simulator is slow; the full length runs on the GPU tier
    frames, warps = make_stream(seed, int(g[case + "_cfg"][2]), n_obj, warp_sigma=3.0 if kind == "botsort" else 0.0)
    res, trk = _run_loop(kind, frames[:n_frames], warps)
    counts = g[case + "_count"]
    off = np.concatenate([[0], np.cumsum(counts)])
    keep = {int(f): i for i, f in enumerate(g[case + "_tlwh_frames"])}
    tl_off = np.concatenate([[0], np.cumsum(counts[g[case + "_tlwh_frames"]])])
    for i in range(n_frames):
        ids = res[i][:, 0].astype(np.int64)
        assert np.array_equal(ids, g[case + "_ids"][off[i]:off[i + 1]]), "track ids differ at frame %d" % (i + 1)
        assert np.array_equal(res[i][:, 5].astype(np.float32), g[case + "_cls"][off[i]:off[i + 1]])
        if i in keep:
            k = keep[i]
            np.testing.assert_allclose(res[i][:, 1:5], g[case + "_tlwh"][tl_off[k]:tl_off[k + 1]], rtol=1e-9, atol=1e-9)


@pytest.mark.parametrize("kind", ["sort", "bytetrack", "botsort"])
def test_fused_step_ignores_boxes_without_area(kind):
    """Detections the reference cannot track -- zero height, non-finite coordinates, and with the xywh filter (BoT-SORT) zero width:
    its Kalman state would turn NaN or its Cholesky factorisation fail -- take no part: the tracks equal those of the stream without
    them, and every output is finite."""
    frames, warps = make_stream(41, 10, 40, warp_sigma=3.0 if kind == "botsort" else 0.0)
    rng = np.random.default_rng(5)
    dirty = [with_flat_boxes(f, rng, xywh=kind == "botsort") for f in frames]
    res, _ = _run_loop(kind, dirty, warps, cap=256, dmax=128)
    orc = T.TrackerOracle(kind)
    for i, f in enumerate(frames):
        exp = orc.update(f, warps[i] if kind == "botsort" else None)
        assert np.isfinite(res[i]).all(), "frame %d" % (i + 1)
        assert [int(v) for v in res[i][:, 0]] == [e[0] for e in exp], "frame %d" % (i + 1)
        if exp:
            np.testing.assert_allclose(res[i][:, 1:5], np.array([e[1] for e in exp]), rtol=1e-9, atol=1e-9)


@pytest.mark.parametrize("kind", ["sort", "bytetrack"])
def test_fused_step_tracks_zero_width_boxes_like_reference(kind):
    """Zero-width, positive-height boxes are defined for the xyah filter and the reference tracks them: the kernel gives the
    reference's ids (tests/golden/refchecks.npz) on every frame and its boxes on the last."""
    g = np.load(os.path.join(GOLDEN, "refchecks.npz"))
    counts = g["flat_%s_count" % kind]
    off = np.concatenate([[0], np.cumsum(counts)])
    frames = zero_width_stream(61, len(counts), 60)
    res, _ = _run_loop(kind, frames, None, cap=256, dmax=128)
    for i in range(len(frames)):
        assert res[i][:, 0].astype(np.int64).tolist() == g["flat_%s_ids" % kind][off[i]:off[i + 1]].tolist(), "frame %d" % (i + 1)
    np.testing.assert_allclose(res[-1][:, 1:5], g["flat_%s_tlwh_last" % kind], rtol=1e-9, atol=1e-9)


def test_fused_step_two_sequences_and_id_base():
    fa, _ = make_stream(21, 12, 30)
    fb, _ = make_stream(22, 12, 45)
    trk = SimTracker("bytetrack", n_seq=2, cap=128, dmax=128, ecap=2048)
    oa, ob = T.TrackerOracle("bytetrack"), T.TrackerOracle("bytetrack")
    for i in range(12):
        r = trk.step([fa[i], fb[i]])
        ea, eb = oa.update(fa[i]), ob.update(fb[i])
        assert [int(v) for v in r[0][:, 0]] == [e[0] for e in ea]
        assert [int(v) for v in r[1][:, 0]] == [e[0] for e in eb]
    # id_base: continue sequence 0's ids from 1000
    r = trk.step([fa[0], fb[0]], id_base=[1000, int(trk.stat[1, L.STAT_NEXT_ID])])
    assert trk.stat[0, L.STAT_NEXT_ID] >= 1000


def test_update_without_detection():
    frames, _ = make_stream(31, 6, 25)
    trk = SimTracker("bytetrack", cap=128, dmax=128, ecap=2048)
    orc = T.TrackerOracle("bytetrack")
    for i in range(4):
        trk.step([frames[i]]); orc.update(frames[i])
    r = trk.step([frames[4]], predict_only=True)[0]
    e = orc.update_without_detection()
    assert [int(v) for v in r[:, 0]] == [x[0] for x in e]
    np.testing.assert_allclose(r[:, 1:5], np.array([x[1] for x in e]), rtol=1e-12, atol=1e-9)


@pytest.mark.parametrize("kind", ["bytetrack", "botsort"])
def test_fused_step_crowded_scene_spills_edges(kind):
    """A crowded scene (300 objects inside a 300 x 300 px area): far more sub-threshold pairs than the shared-memory edge mirror
    holds, so rows live in all three storages -- the mirror, the second window (the idle box arrays) and the global workspace --
    and the augmenting searches run long.  Ids and boxes must still equal the oracle's, frame by frame."""
    frames, warps = make_stream(77, 8, 300, img=700, warp_sigma=2.0 if kind == "botsort" else 0.0)
    trk = SimTracker(kind, cap=1024, dmax=512, ecap=131072)
    orc = T.TrackerOracle(kind)
    most = 0
    for i, f in enumerate(frames):
        w = warps[i].reshape(1, 6) if kind == "botsort" else None
        r = trk.step([f], warps=w)[0]
        e = orc.update(f, warp=warps[i] if kind == "botsort" else None)
        assert trk.stat[0, L.STAT_ERR] == 0
        assert [int(v) for v in r[:, 0]] == [x[0] for x in e], "track ids differ at frame %d" % (i + 1)
        if len(e):
            np.testing.assert_allclose(r[:, 1:5], np.array([x[1] for x in e]), rtol=1e-9, atol=1e-9)
        most = max(most, int(trk.stat[0, 15]))            # stat word 15: sub-threshold pairs of the first association
    assert most > 8000, most
