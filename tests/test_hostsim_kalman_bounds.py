"""not-gpu: the standalone Kalman / IoU entry points of csrc/b2t_tracker.cu (initiate, predict, project, update, gating, gmc_apply,
iou_cost) under the host simulator, in both dtypes and every format, against the extended-precision reference and running error
bound of tests/kalman_ref.py at the edge inputs of tests/kalman_bounds.py; the gating golden of the reference
(tests/golden/kalman_gating.npz); and the proof that these bounds bite: simulator builds with injected bugs, each of which must fail
at the entry point it was made in."""
import ctypes as C
import os
import sys

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "hostsim"))
import build_sim  # noqa: E402
from simlib import ptr, sim  # noqa: E402
from b200track import _lib as L  # noqa: E402
import kalman_bounds as KB  # noqa: E402
import kalman_ref as R  # noqa: E402
import lifecycle_golden as LG  # noqa: E402
import step_bounds as SB  # noqa: E402
from oracle import kalman as K  # noqa: E402

GOLDEN = os.path.join(HERE, "golden")


class SimBackend:
    """The entry points on NumPy arrays through a simulator library."""

    def __init__(self, lib):
        self.lib = lib

    def _c(self, a, dt):
        return np.ascontiguousarray(np.asarray(a, dt))

    def initiate(self, fmt, z):
        f32 = z.dtype == np.float32
        k = len(z)
        mean = np.zeros((k, 8), z.dtype); cov = np.zeros((k, 8, 8), z.dtype)
        L.check(self.lib, self.lib.b2t_kalman_initiate(L.F32 if f32 else L.F64, fmt, ptr(self._c(z, z.dtype)), ptr(mean), ptr(cov), k, None))
        return mean, cov

    def predict(self, fmt, mean, cov, flags, q_f32):
        m, c = mean.copy(), cov.copy()
        L.check(self.lib, self.lib.b2t_kalman_predict(L.F32 if m.dtype == np.float32 else L.F64, fmt, ptr(m), ptr(c),
                                                      ptr(self._c(flags, np.int32)), len(m), int(q_f32), None))
        return m, c

    def project(self, fmt, mean, cov, flags, conf):
        n = len(mean)
        pm = np.zeros((n, 4), mean.dtype); ps = np.zeros((n, 4, 4), mean.dtype)
        cf = None if conf is None else self._c(conf, np.float32)
        L.check(self.lib, self.lib.b2t_kalman_project(L.F32 if mean.dtype == np.float32 else L.F64, fmt, ptr(mean), ptr(cov),
                                                      ptr(self._c(flags, np.int32)), ptr(cf), ptr(pm), ptr(ps), n, None))
        return pm, ps

    def update(self, fmt, mean, cov, idx, z, conf, flags):
        m, c = mean.copy(), cov.copy()
        cf = None if conf is None else self._c(conf, np.float32)
        ix = None if idx is None else self._c(idx, np.int32)
        L.check(self.lib, self.lib.b2t_kalman_update(L.F32 if m.dtype == np.float32 else L.F64, fmt, ptr(m), ptr(c), ptr(ix),
                                                     ptr(self._c(z, m.dtype)), ptr(cf), ptr(self._c(flags, np.int32)), len(z), None))
        return m, c

    def gating(self, fmt, mean, cov, meas, only_position, metric, mean_f32):
        dt = meas.dtype
        out = np.zeros(len(meas), dt)
        L.check(self.lib, self.lib.b2t_kalman_gating(L.F32 if dt == np.float32 else L.F64, fmt, ptr(self._c(mean, dt)), ptr(self._c(cov, dt)),
                                                     ptr(self._c(meas, dt)), len(meas), int(only_position), int(metric),
                                                     L.FLAG_MEAN_F32 if mean_f32 else 0, ptr(out), None))
        return out

    def gmc(self, mean, cov, warp):
        m, c = mean.copy(), cov.copy()
        w6 = (C.c_double * 6)(*np.asarray(warp, np.float64).reshape(-1))
        L.check(self.lib, self.lib.b2t_gmc_apply(L.F32 if m.dtype == np.float32 else L.F64, ptr(m), ptr(c), len(m), w6, None))
        return m, c

    def iou(self, a, b, as_distance):
        n, m = len(a), len(b)
        cost = np.full((n, m), np.nan, a.dtype)
        L.check(self.lib, self.lib.b2t_iou_cost(L.F32 if a.dtype == np.float32 else L.F64, ptr(self._c(a, a.dtype)), n,
                                                ptr(self._c(b, a.dtype)), m, ptr(cost), m, 1, int(as_distance), None))
        return cost


@pytest.fixture(scope="module")
def be():
    return SimBackend(sim())


# n = 128 and n = 4097 run on the GPU only: each simulated thread is a fiber, and 4097 tracks take minutes per entry point here.
# 1, 3, 4, 5, 127 and 129 already cover a lone track, partial groups of the 4-tracks-per-warp mapping and a partial last CTA.
SIM_COUNTS = [1, 3, 4, 5, 127, 129]


# ---------------------------------------------------------------- every entry point, dtype and format
@pytest.mark.parametrize("n", SIM_COUNTS)
@pytest.mark.parametrize("fmt", list(KB.FMTS))
@pytest.mark.parametrize("dtype", ["f32", "f64"])
def test_entry_points_within_bound(be, dtype, fmt, n):
    KB.run_entry_points(be, KB.FMTS[fmt], dtype == "f32", n, seed=1000 * n + 7 * KB.FMTS[fmt] + (dtype == "f32"), stats={})


@pytest.mark.parametrize("fmt", list(KB.FMTS))
@pytest.mark.parametrize("dtype", ["f32", "f64"])
def test_entry_points_bound_is_not_vacuous(be, dtype, fmt):
    """well-conditioned inputs (20 - 300 px, 30 predicts, confidence 0.5): every bound stays below 2^-12 of its magnitude"""
    KB.run_entry_points(be, KB.FMTS[fmt], dtype == "f32", 64, seed=99, stats={}, mild=True)


@pytest.mark.parametrize("n,m", [(1, 1), (5, 129), (130, 257)])
@pytest.mark.parametrize("dtype", ["f32", "f64"])
def test_iou_cost_within_bound(be, dtype, n, m):
    KB.run_iou(be, dtype == "f32", n, m, seed=n * 31 + m, stats={})


def test_f64_kalman_matches_oracle_within_bound(be):
    """float64: the oracle (NumPy / LAPACK, pinned bit for bit to the reference) evaluates the same operations in another order, so
    kernel and oracle both lie within the bound of the exact value: |kernel - oracle| <= 2 x bound"""
    rng = np.random.default_rng(3)
    for name, fmt in KB.FMTS.items():
        mean, cov = KB.states(rng, 33, fmt)
        z = KB.near(rng, mean, fmt).astype(np.float64)
        conf = KB.CONFS[np.arange(33) % 5] if fmt == K.FMT_NSA else None
        um, uc = be.update(fmt, mean, cov, None, z, conf, np.zeros(33, np.int32))
        ms, Ps = R.state(mean, cov, False)
        nm, nP = R.kf_update(ms, Ps, fmt, [R.inputs(z[:, q], False) for q in range(4)], np.zeros(33, bool), conf, False)
        bm, bc = R.bound(R.stack(nm), False), R.bound(R.stack_cov(nP), False)
        for i in range(33):
            om, oc = K.update(fmt, mean[i], cov[i], z[i], False, 0.0 if conf is None else conf[i])
            assert (np.abs(om - um[i]) <= 2 * bm[i]).all(), "%s track %d mean" % (name, i)
            assert (np.abs(oc - uc[i]) <= 2 * bc[i]).all(), "%s track %d cov" % (name, i)


# ---------------------------------------------------------------- the fused step, each frame from its own stored state
class SimStep:
    """The simulator's ctypes tracker with the reads the step check needs (tests/step_bounds.py)."""

    def __init__(self, lib, kind, fmt, dtype, feat_dim=0, **kw):
        self.lib = lib
        self.cfg = L.TrackerConfig(kind=L.KIND_BY_NAME[kind], dtype=dtype, fmt=L.FMT_BY_NAME[fmt], n_seq=1, cap=kw.get("cap", 256),
                                   dmax=kw.get("dmax", 256), ecap=kw.get("ecap", 8192), use_gmc=1, track_buffer=kw.get("track_buffer", 30),
                                   conf_thresh=kw.get("conf_thresh", 0.2), iou_thresh=0.5, frame_rate=kw.get("frame_rate", 30),
                                   feat_dim=feat_dim, theta_iou=0.5, theta_emb=0.25, gamma=0.1)
        nbytes = lib.b2t_tracker_state_bytes(C.byref(self.cfg))
        assert nbytes > 0, lib.b2t_last_error()
        self.mem = np.zeros(nbytes + 256, np.uint8)
        off = (-self.mem.ctypes.data) % 256
        self.h = C.c_void_p()
        L.check(lib, lib.b2t_tracker_create(C.byref(self.cfg), C.c_void_p(self.mem.ctypes.data + off), None, C.byref(self.h)))
        self.cap, self.dmax, self.D = self.cfg.cap, self.cfg.dmax, feat_dim
        self.out = np.zeros((1, self.cap, L.OUT_COLS))
        self.stat = np.zeros((1, L.STAT_WORDS), np.int32)
        if feat_dim:
            self._fbuf = np.zeros(self.dmax * feat_dim + 4, np.float32)
            o = (-self._fbuf.ctypes.data) % 16 // 4
            self.feats = self._fbuf[o:o + self.dmax * feat_dim].reshape(self.dmax, feat_dim)

    def step(self, dets, feats, warp):
        d = np.zeros((1, self.dmax, 6), np.float32)
        a = np.asarray(dets, np.float32).reshape(-1, 6)
        d[0, :len(a)] = a
        cnt = np.array([len(a)], np.int32)
        w = None if warp is None else np.ascontiguousarray(np.asarray(warp, np.float64).reshape(1, 6))
        if self.D:
            self.feats[:] = 0
            self.feats[:len(a)] = feats
            L.check(self.lib, self.lib.b2t_tracker_step_feat(self.h, ptr(d), ptr(cnt), ptr(self.feats), ptr(w), None, ptr(self.out), self.cap,
                                                             ptr(self.stat), 0, None))
        else:
            L.check(self.lib, self.lib.b2t_tracker_step_host(self.h, ptr(d), ptr(cnt), ptr(w), None, ptr(self.out), self.cap,
                                                             ptr(self.stat), 0, None))
        assert self.stat[0, L.STAT_ERR] == 0
        return self.out[0, :self.stat[0, L.STAT_NOUT]].copy()

    def read_slot(self, slot):
        mean = np.zeros(8); cov = np.zeros((8, 8))
        L.check(self.lib, self.lib.b2t_tracker_read_slot(self.h, 0, int(slot), ptr(mean), ptr(cov), None))
        return mean, cov

    def read_list(self, which):
        rows = np.zeros((self.cap + 1, 13))
        n = C.c_int(-1)
        L.check(self.lib, self.lib.b2t_tracker_read_list(self.h, 0, which, ptr(rows), self.cap, C.byref(n), None))
        return rows[:n.value].copy()

    def read_feature(self, slot):
        v = np.zeros(self.D, np.float32)
        L.check(self.lib, self.lib.b2t_tracker_read_feature(self.h, 0, int(slot), ptr(v), None))
        return v


def run_step_case(lib, name, dtype, stats=None):
    kind, fmt, frames, feats, warps, kw = SB.case(name)
    trk = SimStep(lib, kind, fmt, L.F32 if dtype == "f32" else L.F64, **kw)
    return SB.check_stream(trk, frames, warps, kind, L.FMT_BY_NAME[fmt], dtype == "f32", {} if stats is None else stats, name, feats,
                           kw.get("conf_thresh", 0.2))


@pytest.mark.parametrize("name,dtype", SB.step_cases())
def test_step_frames_within_bound(name, dtype):
    counts = run_step_case(sim(), name, dtype)
    assert counts["update"] and counts["birth"] and counts["predict"], counts
    if name.startswith("feat_"):
        assert counts["feature"], counts


# ---------------------------------------------------------------- the bounds bite: injected bugs, each caught where it was made
BUGS = {
    "q_velocity_weight_5pc_f32": ("b2t_kalman.cuh", "const T wgt = pos ? (T)(1.0 / 20) : (T)(1.0 / 160);",
                                  "const T wgt = pos ? (T)(1.0 / 20) : (T)((IsF32<T>::v ? 1.05 : 1.0) / 160);"),
    "gmc_a01_a10_swapped": ("b2t_kalman.cuh", "const T ra = odd ? warp6[3] : warp6[0];   // A[r%2][0]\n    const T rb = odd ? warp6[4] : warp6[1];",
                            "const T ra = odd ? warp6[1] : warp6[0];\n    const T rb = odd ? warp6[4] : warp6[3];"),
    "zero_vh_ignored_f32": ("b2t_kalman.cuh", "if (zero_vh && r == 7) k.m = (T)0;", "if (zero_vh && r == 7 && !IsF32<T>::v) k.m = (T)0;"),
    "nsa_conf_on_variance": ("b2t_kalman.cuh", "if (IsF32<T>::v) return noise_var<T>((T)(omc * (float)s), true);",
                             "if (IsF32<T>::v) return (T)omc * noise_var<T>(s, true);"),
    "iou_height_plus1_dropped_f32": ("b2t_iou.cuh", "const T ih = t_min(a[3], b[3]) - t_max(a[1], b[1]) + (T)1;",
                                     "const T ih = t_min(a[3], b[3]) - t_max(a[1], b[1]) + (T)(sizeof(T) == 4 ? 0 : 1);"),
    # the step's own arithmetic: the first update of a new track without its float32-mean flag (float64 build), a wrong EMA
    # weight on one component of the smoothed feature, the NSA confidence of a matched detection taken as 1 - score
    "first_update_flag_dropped": ("b2t_step.cuh", "f32 = (c.v.flags[slot] & 1) != 0;", "f32 = false;"),
    "ema_weight_off": ("b2t_step.cuh", "r.x = 0.9f * o.x + 0.1f * (a.x / nf);", "r.x = 0.89f * o.x + 0.1f * (a.x / nf);"),
    "nsa_conf_wrong_score": ("b2t_step.cuh", "if (c.p.fmt == FMT_NSA && md == 0) conf = dd[4];", "if (c.p.fmt == FMT_NSA && md == 0) conf = 1.0f - dd[4];"),
    # the output row's x from the mean one velocity step back (the centre before this frame's motion), float build only
    "out_x_stale_mean_f32": ("b2t_step.cuh", "o[1] = (double)box[0];",
                             "o[1] = (double)(IsF32<T>::v ? box[0] - v.mean[(size_t)s * 8 + 4] : box[0]);"),
}


def _variant(name):
    fn, old, new = BUGS[name]
    return L.declare(C.CDLL(build_sim.build_variant(name, [(fn, old, new)])), names=L.TRACKER_SYMBOLS)


@pytest.mark.parametrize("bug,fmt,where", [("q_velocity_weight_5pc_f32", "xyah", "predict"), ("gmc_a01_a10_swapped", "xywh", "gmc"),
                                           ("zero_vh_ignored_f32", "xyah", "predict"), ("nsa_conf_on_variance", "nsa", "project")])
def test_injected_kalman_bug_fails_at_its_entry_point(bug, fmt, where):
    be = SimBackend(_variant(bug))
    with pytest.raises(AssertionError) as e:
        KB.run_entry_points(be, KB.FMTS[fmt], True, 129, seed=11, stats={})
    assert str(e.value).startswith(where), str(e.value)[:300]


def test_injected_iou_bug_fails():
    be = SimBackend(_variant("iou_height_plus1_dropped_f32"))
    KB.run_iou(be, False, 40, 70, seed=3, stats={})                      # the float64 path is untouched
    with pytest.raises(AssertionError, match="^iou_cost f32"):
        KB.run_iou(be, True, 40, 70, seed=3, stats={})


@pytest.mark.parametrize("bug,case,dtype,match", [
    ("out_x_stale_mean_f32", LG.configs()[0], "f32", "frame 2: output rows"),
    ("first_update_flag_dropped", "bytetrack_default", "f64", r"frame \d+: slot \d+ \(id \d+\) is on no path"),
    ("ema_weight_off", "feat_botsort", "f32", r"frame \d+: slot \d+ feature"),
    ("ema_weight_off", "feat_strongsort", "f64", r"frame \d+: slot \d+ feature"),
    ("nsa_conf_wrong_score", "bytetrack_nsa_c03_tb12_fr20", "f32", r"frame \d+: slot \d+ \(id \d+\) is on no path")])
def test_injected_step_bug_fails_at_its_frame(bug, case, dtype, match):
    """each bug fails the frame-by-frame check, and at the first frame its path runs: the same stream on the correct build reaches
    that frame with the check passing"""
    with pytest.raises(AssertionError, match=match) as e:
        run_step_case(_variant(bug), case, dtype)
    frame = int(str(e.value).split(" frame ")[1].split(":")[0])
    kind, fmt, frames, feats, warps, kw = SB.case(case)
    trk = SimStep(sim(), kind, fmt, L.F32 if dtype == "f32" else L.F64, **kw)
    SB.check_stream(trk, frames[:frame], None if warps is None else warps[:frame], kind, L.FMT_BY_NAME[fmt], dtype == "f32", {}, case,
                    None if feats is None else feats[:frame], kw.get("conf_thresh", 0.2))


# ---------------------------------------------------------------- gating against the reference
@pytest.mark.parametrize("name", ["default", "strongsort"])
def test_gating_matches_reference_golden(be, name):
    """the reference's gating_distance on float32 and float64 means (tests/golden/make_golden_gating.py): the oracle and the float64
    kernel at rtol 1e-9, with the float32-mean flag for the float32 means -- without it the noise std is not rounded to float32 and
    the distances move by far more than that"""
    g = np.load(os.path.join(GOLDEN, "kalman_gating.npz"))
    fmt = L.FMT_BY_NAME[name]
    mean, cov, meas, mf = g[name + "_mean"], g[name + "_cov"], g[name + "_meas"].astype(np.float64), g[name + "_mean_f32"]
    assert mf.any() and not mf.all()
    unflagged = 0.0
    for op in (False, True):
        for mi, metric in enumerate(("maha", "gaussian")):
            exp = g["%s_gate_%d_%s" % (name, op, metric)]
            for i in range(len(mean)):
                np.testing.assert_allclose(K.gating_distance(fmt, mean[i], cov[i], meas, op, metric, bool(mf[i])), exp[i], rtol=1e-9)
                got = be.gating(fmt, mean[i], cov[i], meas, op, mi, bool(mf[i]))
                np.testing.assert_allclose(got, exp[i], rtol=1e-9, err_msg="%s state %d only_position=%d %s" % (name, i, op, metric))
                if mf[i] and metric == "maha":
                    old = be.gating(fmt, mean[i], cov[i], meas, op, mi, False)
                    nz = exp[i] > 0
                    unflagged = max(unflagged, float(np.max(np.abs(old - exp[i])[nz] / exp[i][nz])))
    assert unflagged > 1e-8, "the float32-mean states do not tell the two noise roundings apart"
