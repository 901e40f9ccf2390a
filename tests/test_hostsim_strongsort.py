"""not-gpu: StrongSORT on the device (B2T_STRONGSORT) under the fiber simulator.
  * the feature-distance kernel (b2t_feature_distance) against extended-precision distances within the bound tests/featdist_ref.py
    derives, at feat_dim 32 .. 2048, rows / columns 1, 63, 64, 65 and 1024, zero vectors, identical rows, norms 1e-3 and 1e3, with the
    outputs ringed by NaN sentinels -- and the harness failing on injected bugs;
  * the fused step's StrongSORT kind against the reference's goldens (tests/golden/loop_strongsort.npz): ids, tlwh, the tracked and
    lost lists with their states, and the features;
  * a crowded stream whose edges spill past the shared-memory mirror, against the oracle (tests/strongsort_oracle.py)."""
import ctypes as C
import os
import sys

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "hostsim"))
from simlib import ptr, sim  # noqa: E402
from b200track import _lib as L  # noqa: E402
from b200track.synth import make_strongsort_stream  # noqa: E402
import featdist_ref as FR  # noqa: E402
import strongsort_golden as SG  # noqa: E402
from strongsort_oracle import StrongSortOracle  # noqa: E402

PAD = 37


def run_dist(a, b, lib=None):
    """a (B, n, D), b (B, m, D) float32 -> (B, n, m) float64 from b2t_feature_distance, with NaN sentinels checked around it."""
    lib = lib or sim()
    a = np.ascontiguousarray(a, np.float32)
    b = np.ascontiguousarray(b, np.float32)
    B, n, D = a.shape
    m = b.shape[1]
    buf = np.full(B * n * m + 2 * PAD, np.nan)
    L.check(lib, lib.b2t_feature_distance(ptr(a), n, ptr(b), m, D, buf[PAD:].ctypes.data_as(C.c_void_p), B, None))
    assert np.isnan(buf[:PAD]).all() and np.isnan(buf[PAD + B * n * m:]).all(), "a write outside the output"
    return buf[PAD:PAD + B * n * m].reshape(B, n, m)


def _rows(rng, k, D, scale=1.0):
    return (rng.normal(0, 1, (k, D)) * scale / np.sqrt(D)).astype(np.float32)


SHAPES = [(1, 1, 32), (63, 65, 64), (64, 64, 128), (65, 63, 512), (1024, 3, 32), (3, 1024, 32), (9, 7, 2048), (5, 66, 100)]


@pytest.mark.parametrize("n,m,D", SHAPES)
def test_feature_distance_within_bound(n, m, D):
    rng = np.random.default_rng(n * 7919 + m * 31 + D)
    a = np.stack([_rows(rng, n, D), _rows(rng, n, D, 3.0)])
    b = np.stack([_rows(rng, m, D), _rows(rng, m, D, 0.5)])
    got = run_dist(a, b)
    for q in range(2):
        FR.check(got[q], FR.exact(a[q], b[q]), D, "batch %d" % q)


@pytest.mark.parametrize("D", [32, 512, 2048])
def test_feature_distance_special_rows(D):
    rng = np.random.default_rng(D)
    a = np.concatenate([np.zeros((2, D), np.float32), _rows(rng, 4, D), _rows(rng, 3, D, 1e-3), _rows(rng, 3, D, 1e3)])
    b = np.concatenate([np.zeros((1, D), np.float32), a[2:6], _rows(rng, 2, D, 1e-3), _rows(rng, 2, D, 1e3)])
    got = run_dist(a[None], b[None])[0]
    FR.check(got, FR.exact(a, b), D)
    assert (got[:2, 0] == 0).all(), "zero vectors are at distance 0"
    assert (np.diag(got[2:6, 1:5]) == 0).all(), "identical rows are at distance 0"


def test_feature_distance_refuses_bad_arguments():
    lib = sim()
    p = ptr(np.zeros(64, np.float32))
    assert lib.b2t_feature_distance(p, 2, p, 2, 0, p, 1, None) != 0
    assert lib.b2t_feature_distance(p, -1, p, 2, 4, p, 1, None) != 0
    assert lib.b2t_feature_distance(None, 2, p, 2, 4, p, 1, None) != 0


# ---------------------------------------------------------------- the harness catches injected bugs
@pytest.fixture(scope="module")
def case():
    rng = np.random.default_rng(5)
    a, b = _rows(rng, 65, 512), _rows(rng, 63, 512)
    return a, b, run_dist(a[None], b[None])[0]


def test_injected_dropped_k_chunk_fails(case):
    a, b, got = case
    a2, b2 = a.copy(), b.copy()
    a2[:, 16:32] = 0
    b2[:, 16:32] = 0
    with pytest.raises(AssertionError):
        FR.check(got, FR.exact(a2, b2), 512)


def test_injected_shifted_row_fails(case):
    a, b, got = case
    with pytest.raises(AssertionError):
        FR.check(got[1:], FR.exact(a[:-1], b), 512)


def test_injected_missing_clamp_fails(case):
    """the norm-expansion form without max(0, .): a pair of (nearly) identical rows can give the square root of a tiny negative
    number, NaN"""
    a, b, got = case
    bad = got.copy()
    bad[0, 0] = np.nan
    with pytest.raises(AssertionError):
        FR.check(bad, FR.exact(a, b), 512)


def test_injected_bound_one_ulp_tighter_fails(case):
    a, b, got = case
    ex = FR.exact(a, b)
    at = (ex.astype(np.float64) + FR.bound(ex, 512))
    FR.check(np.nextafter(at, 0), ex, 512)                      # just inside the bound: accepted
    with pytest.raises(AssertionError):
        FR.check(np.nextafter(at, np.inf), ex, 512)             # one ulp past it: refused


# ---------------------------------------------------------------- the fused step
class SimStrongSort:
    def __init__(self, n_seq=1, dtype=L.F64, cap=256, dmax=128, ecap=8192, gamma=0.1, fmt="strongsort", track_buffer=30,
                 feat_dim=SG.FEAT_DIM, use_ecc=True):
        lib = sim()
        self.cfg = L.TrackerConfig(kind=L.STRONGSORT, dtype=dtype, fmt=L.FMT_BY_NAME[fmt], n_seq=n_seq, cap=cap, dmax=dmax, ecap=ecap,
                                   use_gmc=int(use_ecc), track_buffer=track_buffer, conf_thresh=0.2, iou_thresh=0.5, frame_rate=30,
                                   feat_dim=feat_dim, theta_iou=0.5, theta_emb=0.25, gamma=gamma)
        nbytes = lib.b2t_tracker_state_bytes(C.byref(self.cfg))
        assert nbytes > 0, lib.b2t_last_error()
        self.mem = np.zeros(nbytes + 256, np.uint8)
        off = (-self.mem.ctypes.data) % 256
        self.h = C.c_void_p()
        L.check(lib, lib.b2t_tracker_create(C.byref(self.cfg), C.c_void_p(self.mem.ctypes.data + off), None, C.byref(self.h)))
        self.S, self.cap, self.dmax, self.D = n_seq, cap, dmax, feat_dim
        self.out = np.zeros((n_seq, cap, L.OUT_COLS))
        self.stat = np.zeros((n_seq, L.STAT_WORDS), np.int32)
        self._fbuf = np.zeros(n_seq * dmax * feat_dim + 4, np.float32)
        o = (-self._fbuf.ctypes.data) % 16 // 4
        self.feats = self._fbuf[o:o + n_seq * dmax * feat_dim].reshape(n_seq, dmax, feat_dim)

    def step(self, dets_list, feats_list, warps=None):
        lib = sim()
        d = np.zeros((self.S, self.dmax, 6), np.float32)
        cnt = np.zeros(self.S, np.int32)
        self.feats[:] = 0
        for s, (a, fe) in enumerate(zip(dets_list, feats_list)):
            d[s, :len(a)] = a
            self.feats[s, :len(a)] = fe
            cnt[s] = len(a)
        w = None if warps is None else np.ascontiguousarray(np.asarray(warps, np.float64).reshape(self.S, 6))
        L.check(lib, lib.b2t_tracker_step_feat(self.h, ptr(d), ptr(cnt), ptr(self.feats), ptr(w), None, ptr(self.out), self.cap,
                                               ptr(self.stat), 0, None))
        return [self.out[s, :self.stat[s, L.STAT_NOUT]].copy() for s in range(self.S)]

    def read_list(self, which, seq=0):
        lib = sim()
        rows = np.zeros((self.cap + 1, 13))
        n = C.c_int(-1)
        L.check(lib, lib.b2t_tracker_read_list(self.h, seq, which, ptr(rows), self.cap, C.byref(n), None))
        return rows[:n.value].copy()

    def read_feature(self, seq, slot):
        v = np.zeros(self.D, np.float32)
        L.check(sim(), sim().b2t_tracker_read_feature(self.h, seq, int(slot), ptr(v), None))
        return v


def _int_rows(rows):
    return rows[:, [0, 8, 9, 11, 12, 10]].astype(np.int64)


def test_config_refusals():
    lib = sim()
    base = dict(kind=L.STRONGSORT, dtype=L.F64, fmt=L.FMT_NSA, n_seq=1, cap=64, dmax=64, ecap=64, use_gmc=1, track_buffer=30,
                conf_thresh=0.2, iou_thresh=0.5, frame_rate=30, feat_dim=64, theta_iou=0.5, theta_emb=0.25, gamma=0.1)
    assert lib.b2t_tracker_state_bytes(C.byref(L.TrackerConfig(**base))) > 0
    for bad in (dict(feat_dim=0), dict(gamma=-0.01), dict(gamma=1.01), dict(gamma=float("nan"))):
        assert lib.b2t_tracker_state_bytes(C.byref(L.TrackerConfig(**dict(base, **bad)))) == 0, bad


@pytest.mark.parametrize("name", [c.name for c in SG.CONFIGS])
def test_strongsort_step_matches_reference(name):
    cfg = next(c for c in SG.CONFIGS if c.name == name).load()
    frames, feats, warps = cfg.stream()
    trk = SimStrongSort(gamma=cfg.gamma, fmt=cfg.fmt, track_buffer=cfg.track_buffer, use_ecc=cfg.use_ecc)
    for i in range(cfg.n_frames):
        where = "%s frame %d" % (name, i + 1)
        res = trk.step([frames[i]], [feats[i]], warps[i].reshape(1, 6) if cfg.use_ecc else None)[0]
        assert trk.stat[0, L.STAT_ERR] == 0, where
        assert res[:, 0].astype(np.int64).tolist() == cfg.ids[i].tolist(), where
        np.testing.assert_allclose(res[:, 1:5], cfg.tlwh[i], rtol=1e-12, atol=1e-9, err_msg=where)
        for w, which in ((0, "tracked"), (1, "lost")):
            assert np.array_equal(_int_rows(trk.read_list(w)), cfg.lists[which][i]), "%s: %s list" % (where, which)
        if i in cfg.feats:
            got = np.array([trk.read_feature(0, s) for s in res[:, 7]]).reshape(len(res), -1)
            np.testing.assert_allclose(got, cfg.feats[i], rtol=0, atol=1e-6, err_msg=where)


def test_strongsort_step_spilled_edges_match_oracle():
    """a crowded stream (300 objects, features close together so that most pairs qualify on appearance): association 1 lists more
    edges than the shared-memory mirror can hold (at most 227 KB / 16 B = 14 528 float64 edges), and the spilled edges must give the
    oracle's ids"""
    frames, feats, warps = make_strongsort_stream(7, 10, 300, 32)
    feats = [(f * 0.2).astype(np.float32) for f in feats]      # distances ~0.06-0.3: every pair under the 0.7 cost
    trk = SimStrongSort(cap=512, dmax=320, ecap=131072, feat_dim=32)
    orc = StrongSortOracle(gamma=0.1)
    spilled = 0
    for i in range(len(frames)):
        res = trk.step([frames[i]], [feats[i]], warps[i].reshape(1, 6))[0]
        exp = orc.update(frames[i], feats[i], warps[i])
        assert trk.stat[0, L.STAT_ERR] == 0
        assert res[:, 0].astype(int).tolist() == [t[0] for t in exp], "frame %d" % (i + 1)
        spilled = max(spilled, int(trk.stat[0, 15]))
    assert spilled > 227 * 1024 // 16, "the stream never spilled past the shared-memory mirror (largest association: %d edges)" % spilled
