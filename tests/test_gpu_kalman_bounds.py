"""-m gpu: the standalone Kalman / IoU entry points (initiate, predict, project, update, gating, gmc_apply, iou_cost) of the nvcc
build on an H100, in both dtypes and every format at n in {1, 3, 4, 5, 127, 128, 129, 4097}, against the extended-precision reference
and running error bound of tests/kalman_ref.py at the edge inputs of tests/kalman_bounds.py; the fused step frame by frame from its
own stored state (tests/step_bounds.py) on every lifecycle configuration and a 4K edge stream; and gating, the drop-in
KalmanFilter / NSAKalmanFilter.gating_distance included, against the reference's golden (tests/golden/kalman_gating.npz).
Prints the largest err / bound per entry point, dtype and format, and per step configuration.  Nothing here reads the reference tree."""
import os
import sys

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

torch = pytest.importorskip("torch")

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
from b200track import _lib as L  # noqa: E402
import kalman_bounds as KB  # noqa: E402
import step_bounds as SB  # noqa: E402
from oracle import kalman as K  # noqa: E402

GOLDEN = os.path.join(HERE, "golden")
TABLE = {}


@pytest.fixture(scope="module")
def ops():
    from b200track.engine import ops as get_ops
    return get_ops()


class GpuBackend:
    def __init__(self, ops):
        self.ops = ops

    def _t(self, a):
        a = np.ascontiguousarray(a)
        return self.ops.dev(a, {np.dtype(np.float32): torch.float32, np.dtype(np.float64): torch.float64, np.dtype(np.int32): torch.int32}[a.dtype])

    @staticmethod
    def _dt(a):
        return L.F32 if a.dtype == np.float32 else L.F64

    def initiate(self, fmt, z):
        m, c = self.ops.kalman_initiate(self._dt(z), fmt, self._t(z))
        return m.cpu().numpy(), c.cpu().numpy()

    def predict(self, fmt, mean, cov, flags, q_f32):
        m, c = self._t(mean), self._t(cov)
        self.ops.kalman_predict(self._dt(mean), fmt, m, c, self._t(flags), q_f32)
        return m.cpu().numpy(), c.cpu().numpy()

    def project(self, fmt, mean, cov, flags, conf):
        pm, ps = self.ops.kalman_project(self._dt(mean), fmt, self._t(mean), self._t(cov), self._t(flags),
                                         None if conf is None else self._t(np.asarray(conf, np.float32)))
        return pm.cpu().numpy(), ps.cpu().numpy()

    def update(self, fmt, mean, cov, idx, z, conf, flags):
        m, c = self._t(mean), self._t(cov)
        self.ops.kalman_update(self._dt(mean), fmt, m, c, self._t(z), None if idx is None else self._t(np.asarray(idx, np.int32)),
                               None if conf is None else self._t(np.asarray(conf, np.float32)), self._t(flags))
        return m.cpu().numpy(), c.cpu().numpy()

    def gating(self, fmt, mean, cov, meas, only_position, metric, mean_f32):
        dt = meas.dtype
        return self.ops.kalman_gating(self._dt(meas), fmt, self._t(np.asarray(mean, dt)), self._t(np.asarray(cov, dt)), self._t(meas),
                                      only_position, metric, mean_f32).cpu().numpy()

    def gmc(self, mean, cov, warp):
        m, c = self._t(mean), self._t(cov)
        self.ops.gmc_apply(self._dt(mean), m, c, warp)
        return m.cpu().numpy(), c.cpu().numpy()

    def iou(self, a, b, as_distance):
        return self.ops.iou_cost(self._dt(a), self._t(a), self._t(b), bool(as_distance)).cpu().numpy()


@pytest.mark.parametrize("fmt", list(KB.FMTS))
@pytest.mark.parametrize("dtype", ["f32", "f64"])
def test_entry_points_within_bound(ops, dtype, fmt):
    be = GpuBackend(ops)
    stats = {}
    for n in KB.COUNTS:
        KB.run_entry_points(be, KB.FMTS[fmt], dtype == "f32", n, seed=1000 * n + 7 * KB.FMTS[fmt] + (dtype == "f32"), stats=stats)
    KB.run_entry_points(be, KB.FMTS[fmt], dtype == "f32", 64, seed=99, stats={}, mild=True)
    KB.run_iou(be, dtype == "f32", 129, 257, seed=5 + KB.FMTS[fmt], stats=stats)
    TABLE[(dtype, fmt)] = stats
    print("\nlargest err/bound %s %s: %s" % (dtype, fmt, ", ".join("%s %.3f" % kv for kv in sorted(stats.items()))))


@pytest.mark.parametrize("name,dtype", SB.step_cases())
def test_step_frames_within_bound(name, dtype):
    from b200track.engine import TrackEngine
    kind, fmt, frames, feats, warps, kw = SB.case(name)
    eng = TrackEngine(kind, n_seq=1, dtype=dtype, cap=256, dmax=256, kalman_format=fmt, device="cuda:0", **kw)

    class Adapter:
        def step(self, dets, fe, warp):
            w = None if warp is None else np.asarray(warp).reshape(1, 6)
            d = torch.as_tensor(np.asarray(dets, np.float32).reshape(-1, 6), device="cuda:0")
            if fe is None:
                return eng.step_cuda_dets([d], w)[0].copy()
            f = torch.as_tensor(np.ascontiguousarray(fe, np.float32), device="cuda:0")
            return eng.step_cuda_dets([d], w, feats_list=[f])[0].copy()

        def read_slot(self, slot):
            return eng.read_slot(0, slot)

        def read_list(self, which):
            return eng.read_list(0, "tracked" if which == 0 else "lost")

        def read_feature(self, slot):
            return eng.read_feature(0, slot)

    stats = {}
    counts = SB.check_stream(Adapter(), frames, warps, kind, L.FMT_BY_NAME[fmt], dtype == "f32", stats, name, feats,
                             kw.get("conf_thresh", 0.2))
    assert counts["update"] and counts["birth"] and counts["predict"], counts
    if feats is not None:
        assert counts["feature"], counts
    print("\nlargest err/bound step %s %s: %s (checked: %s)" % (
        name, dtype, ", ".join("%s %.3f" % kv for kv in sorted(stats.items())), ", ".join("%s %d" % kv for kv in sorted(counts.items()))))


@pytest.mark.parametrize("name", ["default", "strongsort"])
def test_gating_and_dropin_match_reference_golden(ops, name):
    """the float64 kernel and the drop-in gating_distance (which passes the mean's dtype on) against the reference at rtol 1e-9"""
    sys.path.insert(0, os.path.join(os.path.dirname(HERE), "yolov7-tracker_b200", "tracker"))
    import kalman_filter as KF                                      # the drop-in, by its bare name as track.py imports it
    kf = KF.KalmanFilter() if name == "default" else KF.NSAKalmanFilter()
    g = np.load(os.path.join(GOLDEN, "kalman_gating.npz"))
    fmt = L.FMT_BY_NAME[name]
    be = GpuBackend(ops)
    mean, cov, meas, mf = g[name + "_mean"], g[name + "_cov"], g[name + "_meas"].astype(np.float64), g[name + "_mean_f32"]
    for op in (False, True):
        for mi, metric in enumerate(("maha", "gaussian")):
            exp = g["%s_gate_%d_%s" % (name, op, metric)]
            for i in range(len(mean)):
                where = "%s state %d only_position=%d %s" % (name, i, op, metric)
                np.testing.assert_allclose(be.gating(fmt, mean[i], cov[i], meas, op, mi, bool(mf[i])), exp[i], rtol=1e-9, err_msg=where)
                m_in = mean[i].astype(np.float32) if mf[i] else mean[i]
                np.testing.assert_allclose(kf.gating_distance(m_in, cov[i], meas, op, metric), exp[i], rtol=1e-9, err_msg="drop-in " + where)


def test_botsort_dropin_gating_within_bound(ops):
    """the reference's BoT-SORT filter has no gating_distance; the drop-in's extra one is held to the bound"""
    sys.path.insert(0, os.path.join(os.path.dirname(HERE), "yolov7-tracker_b200", "tracker"))
    import kalman_filter as KF                                      # the drop-in, by its bare name as track.py imports it
    import kalman_ref as R
    kf = KF.BoTSORTKalmanFilter()
    rng = np.random.default_rng(8)
    mean, cov = KB.states(rng, 4, K.FMT_XYWH)
    meas = KB.near(rng, mean, K.FMT_XYWH, 3.0).astype(np.float64)
    for i in range(4):
        for mean_f32 in (False, True):
            for op in (False, True):
                for mi, metric in enumerate(("maha", "gaussian")):
                    m_in = mean[i].astype(np.float32) if mean_f32 else mean[i]
                    ref = R.gating(K.FMT_XYWH, m_in.astype(np.float64), cov[i], meas, op, mi, False, mean_f32)
                    R.check(kf.gating_distance(m_in, cov[i], meas, op, metric), ref, False, "botsort drop-in gating %d" % i)
