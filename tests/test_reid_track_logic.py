"""not-gpu: BoT-SORT with appearance features.  The oracle (tests/reid_track_oracle.py) against the unmodified reference's outputs
(tests/golden/loop_botsort_reid.npz), and the fused step's feature path (b2t_tracker_step_feat, csrc/b2t_step.cuh) executed by the
fiber simulator against the oracle.  The nvcc build runs the same checks on an H100 in tests/test_gpu_reid_track.py."""
import ctypes as C
import os
import sys

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "hostsim"))
sys.path.insert(0, HERE)
from simlib import ptr, sim  # noqa: E402
from b200track import _lib as L  # noqa: E402
from b200track.synth import make_reid_stream  # noqa: E402
from oracle import trackers as T  # noqa: E402
from reid_track_oracle import ReidBotsortOracle  # noqa: E402

GOLDEN = os.path.join(HERE, "golden")
EINVAL = -1                     # B2T_EINVAL


def _golden():
    g = np.load(os.path.join(GOLDEN, "loop_botsort_reid.npz"))
    seed, n_obj, n_frames, dim = [int(v) for v in g["cfg"]]
    frames, feats, warps = make_reid_stream(seed, n_frames, n_obj, dim)
    return g, frames, feats, warps


def _split(g):
    off = np.concatenate([[0], np.cumsum(g["count"])])
    fk = {int(f): i for i, f in enumerate(g["feat_frames"])}
    foff = np.concatenate([[0], np.cumsum(g["count"][g["feat_frames"]])])
    return off, fk, foff


def test_oracle_equals_reference_golden_bit_for_bit():
    g, frames, feats, warps = _golden()
    from b200track.synth import stream_digest
    assert stream_digest(frames) == str(g["digest"]) and stream_digest(feats) == str(g["feat_digest"])
    off, fk, foff = _split(g)
    orc = ReidBotsortOracle()
    for i, (f, fe) in enumerate(zip(frames, feats)):
        exp = orc.update(f, warps[i], feats=fe)
        assert np.array_equal(np.array([e[0] for e in exp], np.int32), g["ids"][off[i]:off[i + 1]]), "ids differ at frame %d" % (i + 1)
        assert np.array_equal(np.array([e[1] for e in exp]).reshape(-1, 4), g["tlwh"][off[i]:off[i + 1]]), "tlwh differ at frame %d" % (i + 1)
        if i in fk:
            k = fk[i]
            assert np.array_equal(orc.last_features(), g["feats"][foff[k]:foff[k + 1]]), "features differ at frame %d" % (i + 1)


def test_oracle_without_features_is_the_iou_botsort_oracle():
    frames, _, warps = make_reid_stream(5, 30, 40, 32)
    a, b = ReidBotsortOracle(), T.TrackerOracle("botsort")
    for i, f in enumerate(frames):
        ea, eb = a.update(f, warps[i]), b.update(f, warps[i])
        assert [e[0] for e in ea] == [e[0] for e in eb]
        assert all(np.array_equal(x[1], y[1]) for x, y in zip(ea, eb))


def _cfg(kind="botsort", dtype=L.F64, cap=256, dmax=256, ecap=8192, feat_dim=64, theta_iou=0.5, theta_emb=0.25):
    return L.TrackerConfig(kind=L.KIND_BY_NAME[kind], dtype=dtype, fmt=L.FMT_BY_NAME["botsort" if kind == "botsort" else "default"],
                           n_seq=1, cap=cap, dmax=dmax, ecap=ecap, use_gmc=1, track_buffer=30, conf_thresh=0.2, iou_thresh=0.5,
                           frame_rate=30, feat_dim=feat_dim, theta_iou=theta_iou, theta_emb=theta_emb)


class SimFeatTracker:
    """b2t_tracker_step_feat on simulator memory (NumPy arrays stand in for device memory)."""

    def __init__(self, **kw):
        lib = sim()
        self.cfg = _cfg(**kw)
        nbytes = lib.b2t_tracker_state_bytes(C.byref(self.cfg))
        assert nbytes > 0, lib.b2t_last_error()
        self.mem = np.zeros(nbytes + 256, np.uint8)
        off = (-self.mem.ctypes.data) % 256
        self.h = C.c_void_p()
        L.check(lib, lib.b2t_tracker_create(C.byref(self.cfg), C.c_void_p(self.mem.ctypes.data + off), None, C.byref(self.h)))
        self.D, self.dmax, self.cap = self.cfg.feat_dim, self.cfg.dmax, self.cfg.cap
        self.out = np.zeros((1, self.cap, L.OUT_COLS), np.float64)
        self.stat = np.zeros((1, L.STAT_WORDS), np.int32)

    def step(self, dets, feats, warp):
        lib = sim()
        d = np.zeros((1, self.dmax, 6), np.float32)
        d[0, :len(dets)] = dets
        fe = np.zeros((1, self.dmax, self.D), np.float32)
        fe[0, :len(dets)] = feats
        cnt = np.array([len(dets)], np.int32)
        w = np.ascontiguousarray(np.asarray(warp, np.float64).reshape(1, 6))
        L.check(lib, lib.b2t_tracker_step_feat(self.h, ptr(d), ptr(cnt), ptr(fe), ptr(w), None, ptr(self.out), self.cap,
                                               ptr(self.stat), 0, None))
        assert self.stat[0, L.STAT_ERR] == 0
        return self.out[0, :self.stat[0, L.STAT_NOUT]].copy()

    def feature(self, slot):
        v = np.zeros(self.D, np.float32)
        L.check(sim(), sim().b2t_tracker_read_feature(self.h, 0, int(slot), ptr(v), None))
        return v


def test_hostsim_step_feat_matches_oracle():
    """The kernel's feature path on the reference-pinned stream: ids and boxes as the oracle, features within 1e-6."""
    g, frames, feats, warps = _golden()
    n_frames = 32                 # the simulator is slow; the full stream runs on the GPU tier
    trk, orc = SimFeatTracker(feat_dim=int(g["cfg"][3])), ReidBotsortOracle()
    napp = nlow = 0
    for i in range(n_frames):
        got = trk.step(frames[i], feats[i], warps[i])
        exp = orc.update(frames[i], warps[i], feats=feats[i])
        assert [int(v) for v in got[:, 0]] == [e[0] for e in exp], "ids differ at frame %d" % (i + 1)
        np.testing.assert_allclose(got[:, 1:5], np.array([e[1] for e in exp]).reshape(-1, 4), rtol=1e-9, atol=1e-9)
        ef = orc.last_features()
        for k, row in enumerate(got):
            np.testing.assert_allclose(trk.feature(row[7]), ef[k], rtol=0, atol=1e-6)
        napp += trk.stat[0, L.STAT_NAPP]
        nlow += trk.stat[0, L.STAT_NAPPLOW]
    assert napp > 0 and 0 < nlow <= napp


def test_hostsim_feature_abi_checks():
    lib = sim()
    size = lambda **kw: lib.b2t_tracker_state_bytes(C.byref(_cfg(**kw)))     # noqa: E731
    # feat_dim = 0 is today's tracker: same state size whatever the theta fields hold
    assert size(feat_dim=0) == size(feat_dim=0, theta_iou=3.0, theta_emb=-1.0) > 0
    assert size(feat_dim=512) > size(feat_dim=0)
    # the C4 configuration keeps working with 512-d features (they live in device memory, not shared memory)
    assert lib.b2t_tracker_state_bytes(C.byref(_cfg(cap=1152, dmax=576, ecap=147456, feat_dim=512))) > 0
    for bad in (dict(kind="bytetrack"), dict(feat_dim=48), dict(feat_dim=4096), dict(feat_dim=-32), dict(theta_iou=1.0),
                dict(theta_iou=1.5), dict(theta_iou=float("nan"))):
        assert size(**bad) == 0, bad
    mem = np.zeros(size(feat_dim=64) + 256, np.uint8)
    h = C.c_void_p()
    base = C.c_void_p(mem.ctypes.data + (-mem.ctypes.data) % 256)
    L.check(lib, lib.b2t_tracker_create(C.byref(_cfg(feat_dim=64)), base, None, C.byref(h)))
    d = np.zeros((1, 256, 6), np.float32)
    fe = np.zeros((1, 256, 64), np.float32)
    cnt = np.zeros(1, np.int32)
    out = np.zeros((1, 256, 8))
    st = np.zeros((1, 64), np.int32)
    assert lib.b2t_tracker_step(h, ptr(d), ptr(cnt), None, None, ptr(out), 256, ptr(st), 0, None) == EINVAL
    assert lib.b2t_tracker_step_feat(h, ptr(d), ptr(cnt), None, None, None, ptr(out), 256, ptr(st), 0, None) == EINVAL
    assert lib.b2t_tracker_set_thetas(h, 1.0, 0.25) == EINVAL
    assert lib.b2t_tracker_set_thetas(h, 0.4, 0.3) == 0
    lib.b2t_tracker_destroy(h)
    h2 = C.c_void_p()
    mem2 = np.zeros(size(feat_dim=0) + 256, np.uint8)
    L.check(lib, lib.b2t_tracker_create(C.byref(_cfg(feat_dim=0)), C.c_void_p(mem2.ctypes.data + (-mem2.ctypes.data) % 256), None, C.byref(h2)))
    assert lib.b2t_tracker_step_feat(h2, ptr(d), ptr(cnt), ptr(fe), None, None, ptr(out), 256, ptr(st), 0, None) == EINVAL
    v = np.zeros(64, np.float32)
    assert lib.b2t_tracker_read_feature(h2, 0, 0, ptr(v), None) == EINVAL
    lib.b2t_tracker_destroy(h2)


@pytest.mark.parametrize("theta_iou, theta_emb", [(0.3, 0.25), (0.5, 0.1)])
def test_hostsim_thetas_follow_the_attributes(theta_iou, theta_emb):
    frames, feats, warps = make_reid_stream(9, 12, 30, 32)
    trk, orc = SimFeatTracker(feat_dim=32), ReidBotsortOracle(theta_iou=theta_iou, theta_emb=theta_emb)
    L.check(sim(), sim().b2t_tracker_set_thetas(trk.h, theta_iou, theta_emb))
    for i in range(len(frames)):
        got = trk.step(frames[i], feats[i], warps[i])
        exp = orc.update(frames[i], warps[i], feats=feats[i])
        assert [int(v) for v in got[:, 0]] == [e[0] for e in exp]
