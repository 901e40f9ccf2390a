"""not-gpu: UAVMOT on the device (B2T_UAVMOT) under the fiber simulator.
  * the fused step's UAVMOT kind against the reference's goldens (tests/golden/loop_uavmot.npz): ids, tlwh and the tracked and lost
    lists with their states;
  * a 300-object stream against the oracle (tests/uavmot_oracle.py);
  * b2t_structure_vectors / b2t_structure_distance against the oracle at their edges, and the harness failing on injected bugs
    (last-index ties, <= 400, S dropped, the fused cost read from the wrong row, the first solve's matches kept, q20 ignored,
    q21 "fixed"), and float32 refused for this kind."""
import ctypes as C
import os
import sys

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "hostsim"))
import build_sim  # noqa: E402
from simlib import SimTracker, ptr, sim  # noqa: E402
from b200track import _lib as L  # noqa: E402
from b200track.synth import make_stream  # noqa: E402
import uavmot_golden as UG  # noqa: E402
import uavmot_oracle as U  # noqa: E402


def read_list(lib, trk, which):
    rows = np.zeros((trk.cap + 1, 13))
    n = C.c_int(-1)
    L.check(lib, lib.b2t_tracker_read_list(trk.h, 0, which, ptr(rows), trk.cap, C.byref(n), None))
    return rows[:n.value, [0, 8, 9, 11, 12, 10]].astype(np.int64)


def run_golden(cfg, lib=None):
    """Runs the config through a simulator build; returns the first mismatch, or None."""
    lib = lib or sim()
    trk = SimTracker(kind="uavmot", kalman_format=cfg.fmt, track_buffer=cfg.track_buffer, cap=256, dmax=128)
    if lib is not sim():
        trk = _SimOn(lib, cfg)
    for i, fr in enumerate(cfg.stream()):
        res = trk.step([fr])[0]
        if res[:, 0].astype(np.int64).tolist() != cfg.ids[i].tolist():
            return "frame %d: ids" % (i + 1)
        if not np.allclose(res[:, 1:5], cfg.tlwh[i], rtol=1e-12, atol=1e-9):
            return "frame %d: tlwh" % (i + 1)
        for w, which in ((0, "tracked"), (1, "lost")):
            if not np.array_equal(read_list(lib, trk, w), cfg.lists[which][i]):
                return "frame %d: %s list" % (i + 1, which)
    return None


class _SimOn(SimTracker):
    """SimTracker on another simulator build (an injected bug)"""

    def __init__(self, lib, cfg):
        self.lib = lib
        self.cfg = L.TrackerConfig(kind=L.UAVMOT, dtype=L.F64, fmt=L.FMT_BY_NAME[cfg.fmt], n_seq=1, cap=256, dmax=128, ecap=8192,
                                   use_gmc=0, track_buffer=cfg.track_buffer, conf_thresh=0.2, iou_thresh=0.5, frame_rate=30)
        nbytes = lib.b2t_tracker_state_bytes(C.byref(self.cfg))
        self.mem = np.zeros(nbytes + 256, np.uint8)
        off = (-self.mem.ctypes.data) % 256
        self.h = C.c_void_p()
        L.check(lib, lib.b2t_tracker_create(C.byref(self.cfg), C.c_void_p(self.mem.ctypes.data + off), None, C.byref(self.h)))
        self.S, self.cap, self.dmax = 1, 256, 128
        self.out = np.zeros((1, 256, L.OUT_COLS))
        self.stat = np.zeros((1, L.STAT_WORDS), np.int32)

    def step(self, dets_list):
        d = np.zeros((1, self.dmax, 6), np.float32)
        a = np.asarray(dets_list[0], np.float32).reshape(-1, 6)
        d[0, :len(a)] = a
        cnt = np.array([len(a)], np.int32)
        L.check(self.lib, self.lib.b2t_tracker_step_host(self.h, ptr(d), ptr(cnt), None, None, ptr(self.out), self.cap, ptr(self.stat),
                                                         0, None))
        return [self.out[0, :self.stat[0, L.STAT_NOUT]].copy()]


@pytest.mark.parametrize("name", [c.name for c in UG.CONFIGS])
def test_uavmot_step_matches_reference(name):
    cfg = next(c for c in UG.CONFIGS if c.name == name).load()
    assert run_golden(cfg) is None


def test_uavmot_step_300_objects_matches_oracle():
    frames, _ = make_stream(21, 12, n_obj=300)
    trk = SimTracker(kind="uavmot", cap=1024, dmax=400, ecap=65536)
    orc = U.UavmotOracle()
    for i, fr in enumerate(frames):
        res = trk.step([fr])[0]
        exp = orc.update(fr)
        assert trk.stat[0, L.STAT_ERR] == 0
        assert res[:, 0].astype(int).tolist() == [t[0] for t in exp], "frame %d" % (i + 1)
        np.testing.assert_allclose(res[:, 1:5], np.array([t[1] for t in exp]).reshape(-1, 4), rtol=1e-12, atol=1e-9)


def structure_vectors(lib, pts, detection):
    pts = np.ascontiguousarray(pts, np.float32 if detection else np.float64).reshape(-1, 2)
    out = np.full((len(pts) + 2, 3), np.nan)
    L.check(lib, lib.b2t_structure_vectors(L.F32 if detection else L.F64, ptr(pts), len(pts), ptr(out[1:]), None))
    assert np.isnan(out[0]).all() and np.isnan(out[-1]).all(), "a write outside the output"
    return out[1:-1]


def structure_distance(lib, a, b):
    a = np.ascontiguousarray(a, np.float64)
    b = np.ascontiguousarray(b, np.float64)
    out = np.zeros((len(a), len(b)))
    L.check(lib, lib.b2t_structure_distance(ptr(a), len(a), ptr(b), len(b), ptr(out), None))
    return out


def edge_sets():
    rng = np.random.default_rng(9)
    lattice = rng.integers(0, 9, (40, 2)).astype(np.float64) * 100             # ties, 400 exactly, axes and diagonals
    return [np.zeros((0, 2)), np.array([[3.0, 4.0]]), np.full((7, 2), 11.0), np.array([[0, 0], [400, 0], [0, 399.5], [-250, 250]]),
            lattice, lattice + rng.integers(-1, 2, lattice.shape), rng.uniform(-50, 1300, (200, 2))]


def check_structure(lib):
    for pts in edge_sets():
        for det in (False, True):
            got = structure_vectors(lib, pts, det)
            want = U.structure_vectors(pts.astype(np.float32) if det else pts, det)
            if not np.array_equal(got, want):
                return "vectors (detection=%s, n=%d)" % (det, len(pts))
        a = U.structure_vectors(pts)
        b = U.structure_vectors(pts.astype(np.float32), True)
        if len(a) and not np.array_equal(structure_distance(lib, a, b), U.structure_distance(a, b)):
            return "distance (n=%d)" % len(pts)
    return None


def test_structure_entries_match_oracle():
    assert check_structure(sim()) is None


def test_float32_is_refused():
    lib = sim()
    for dtype, ok in ((L.F64, True), (L.F32, False)):
        cfg = L.TrackerConfig(kind=L.UAVMOT, dtype=dtype, fmt=L.FMT_XYAH, n_seq=1, cap=64, dmax=64, ecap=64, use_gmc=0, track_buffer=30,
                              conf_thresh=0.2, iou_thresh=0.5, frame_rate=30)
        assert (lib.b2t_tracker_state_bytes(C.byref(cfg)) > 0) == ok
    assert b"F64" in lib.b2t_last_error()


def test_structure_entries_refuse_bad_arguments():
    lib = sim()
    p = ptr(np.zeros(8))
    assert lib.b2t_structure_vectors(L.F64, p, -1, p, None) != 0
    assert lib.b2t_structure_vectors(7, p, 2, p, None) != 0
    assert lib.b2t_structure_distance(None, 2, p, 2, p, None) != 0


STEP = "b2t_step.cuh"
BUGS = {
    "last_index_ties": ([(STEP, "if (imax < 0 || l > lmax) { lmax = l; imax = j; }", "if (imax < 0 || l >= lmax) { lmax = l; imax = j; }"),
                         (STEP, "if (oi >= 0 && (imax < 0 || ol > lmax || (ol == lmax && oi < imax)))",
                          "if (oi >= 0 && (imax < 0 || ol > lmax || (ol == lmax && oi > imax)))")], "structure"),
    "le_400": ([(STEP, "if (l < (P)UAV_LOCAL_R && l > (P)0)", "if (l <= (P)UAV_LOCAL_R && l > (P)0)")], "structure"),
    "q20_ignored": ([(STEP, "return x0[i] >= 0 && (i != 0 || x0[i] != 0);", "return x0[i] >= 0;")], "golden"),
    "s_dropped": ([(STEP, "(1.0 - UAV_LAMBDA) * uav_struct_dist(app->sv_row + 3 * i, app->sv_col + 3 * j)", "(1.0 - UAV_LAMBDA) * 0.0")], "golden"),
    "s_row0": ([(STEP, "uav_struct_dist(app->sv_row + 3 * i, app->sv_col + 3 * j)", "uav_struct_dist(app->sv_row, app->sv_col + 3 * j)")], "golden"),
    "first_solve_kept": ([(STEP, "            if (any > 0) {", "            if (any > 0 && false) {")], "golden"),
    "q21_fixed": ([(STEP, "if (x[k] < 0) { v.state[sm.pool[k]] = ST_LOST; sm.dupa[k] |= 8; }",
                    "if (x[k] < 0) { v.state[sm.nlo[k]] = ST_LOST; sm.dupa[sm.ut[k]] |= 8; }")], "golden"),
}


@pytest.mark.parametrize("bug", sorted(BUGS))
def test_injected_bug_fails(bug):
    patches, where = BUGS[bug]
    lib = L.declare(C.CDLL(build_sim.build_variant("uav_" + bug, patches)), names=L.TRACKER_SYMBOLS)
    if where == "structure":
        assert check_structure(lib) is not None, "the structure harness did not notice %s" % bug
    else:
        assert any(run_golden(c.load(), lib) is not None for c in UG.CONFIGS), "the goldens did not notice %s" % bug
