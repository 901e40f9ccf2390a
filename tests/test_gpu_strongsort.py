"""gpu: StrongSORT on the H100 (TrackEngine("strongsort"), B2T_STRONGSORT).
  * the reference's goldens (tests/golden/loop_strongsort.npz): ids exact, tlwh within 1e-9, lists exact, features within 1e-6;
  * four different sequences in one launch give bitwise the results of each sequence alone;
  * the float32 engine keeps the ids of the float64 one;
  * a C4-sized stream (300 objects, 512-d features) against the oracle: ids exact;
  * the feature-distance kernel against extended precision within its derived bound, at the simulator's cases and at
    1024 x 1024 x 512 x 8 sequences."""
import ctypes as C
import os
import sys

import numpy as np
import pytest

pytestmark = pytest.mark.gpu
torch = pytest.importorskip("torch")

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
from b200track import _lib as L                                # noqa: E402
from b200track.synth import make_strongsort_stream             # noqa: E402
import featdist_ref as FR                                      # noqa: E402
import strongsort_golden as SG                                 # noqa: E402
from strongsort_oracle import StrongSortOracle                 # noqa: E402


def _engine(n_seq=1, dtype="f64", cap=256, dmax=128, feat_dim=SG.FEAT_DIM, **kw):
    from b200track.engine import TrackEngine
    return TrackEngine("strongsort", n_seq=n_seq, dtype=dtype, cap=cap, dmax=dmax, feat_dim=feat_dim, **kw)


def _step(eng, frames, feats, warps=None):
    dl = [torch.as_tensor(f).cuda() for f in frames]
    fl = [torch.as_tensor(f).cuda() for f in feats]
    return [r.copy() for r in eng.step_cuda_dets(dl, warps=warps, feats_list=fl)]


def _int_rows(rows):
    return rows[:, [0, 8, 9, 11, 12, 10]].astype(np.int64)


@pytest.mark.parametrize("name", [c.name for c in SG.CONFIGS])
def test_engine_matches_reference(name):
    cfg = next(c for c in SG.CONFIGS if c.name == name).load()
    frames, feats, warps = cfg.stream()
    eng = _engine(gamma=cfg.gamma, kalman_format=cfg.fmt, track_buffer=cfg.track_buffer, use_gmc=cfg.use_ecc)
    for i in range(cfg.n_frames):
        where = "%s frame %d" % (name, i + 1)
        res = _step(eng, [frames[i]], [feats[i]], warps[i].reshape(1, 6) if cfg.use_ecc else None)[0]
        assert res[:, 0].astype(np.int64).tolist() == cfg.ids[i].tolist(), where
        np.testing.assert_allclose(res[:, 1:5], cfg.tlwh[i], rtol=0, atol=1e-9, err_msg=where)
        for which in ("tracked", "lost"):
            assert np.array_equal(_int_rows(eng.read_list(0, which)), cfg.lists[which][i]), "%s: %s list" % (where, which)
        if i in cfg.feats:
            got = np.array([eng.read_feature(0, s) for s in res[:, 7]]).reshape(len(res), -1)
            np.testing.assert_allclose(got, cfg.feats[i], rtol=0, atol=1e-6, err_msg=where)


def test_four_sequences_in_one_launch_equal_each_alone():
    streams = [make_strongsort_stream(100 + q, 60, 40 + 10 * q, SG.FEAT_DIM) for q in range(4)]
    eng = _engine(n_seq=4)
    alone = [_engine() for _ in range(4)]
    for i in range(60):
        w = np.stack([s[2][i] for s in streams]).reshape(4, 6)
        both = _step(eng, [s[0][i] for s in streams], [s[1][i] for s in streams], w)
        for q in range(4):
            one = _step(alone[q], [streams[q][0][i]], [streams[q][1][i]], w[q:q + 1])[0]
            assert np.array_equal(both[q], one), "sequence %d frame %d" % (q, i + 1)


def test_float32_engine_keeps_the_ids():
    cfg = SG.CONFIGS[0].load()
    frames, feats, warps = cfg.stream()
    eng = _engine(dtype="f32", gamma=cfg.gamma)
    for i in range(cfg.n_frames):
        res = _step(eng, [frames[i]], [feats[i]], warps[i].reshape(1, 6))[0]
        assert res[:, 0].astype(np.int64).tolist() == cfg.ids[i].tolist(), "frame %d" % (i + 1)
        np.testing.assert_allclose(res[:, 1:5], cfg.tlwh[i], rtol=1e-4, atol=2e-2, err_msg="frame %d" % (i + 1))


def test_c4_sized_stream_matches_oracle():
    frames, feats, warps = make_strongsort_stream(11, 60, 300, 512)
    eng = _engine(cap=1024, dmax=512, feat_dim=512)
    orc = StrongSortOracle(gamma=0.1)
    for i in range(len(frames)):
        res = _step(eng, [frames[i]], [feats[i]], warps[i].reshape(1, 6))[0]
        exp = orc.update(frames[i], feats[i], warps[i])
        assert res[:, 0].astype(int).tolist() == [t[0] for t in exp], "frame %d" % (i + 1)


def _dist(a, b):
    lib = L.load()
    a_t, b_t = torch.as_tensor(a).cuda().contiguous(), torch.as_tensor(b).cuda().contiguous()
    B, n, D = a.shape
    m = b.shape[1]
    buf = torch.full((B * n * m + 64,), float("nan"), dtype=torch.float64, device="cuda")
    L.check(lib, lib.b2t_feature_distance(C.c_void_p(a_t.data_ptr()), n, C.c_void_p(b_t.data_ptr()), m, D,
                                          C.c_void_p(buf.data_ptr() + 32 * 8), B, C.c_void_p(torch.cuda.current_stream().cuda_stream)))
    out = buf.cpu().numpy()
    assert np.isnan(out[:32]).all() and np.isnan(out[32 + B * n * m:]).all()
    return out[32:32 + B * n * m].reshape(B, n, m)


SHAPES = [(1, 1, 32), (63, 65, 64), (64, 64, 128), (65, 63, 512), (1024, 3, 32), (3, 1024, 32), (9, 7, 2048), (5, 66, 100)]


@pytest.mark.parametrize("n,m,D", SHAPES)
def test_feature_distance_within_bound(n, m, D):
    rng = np.random.default_rng(n * 7919 + m * 31 + D)
    a = (rng.normal(0, 1, (2, n, D)) / np.sqrt(D)).astype(np.float32)
    b = (rng.normal(0, 1, (2, m, D)) / np.sqrt(D)).astype(np.float32)
    a[1] *= 1e3
    b[1] *= 1e-3
    got = _dist(a, b)
    for q in range(2):
        FR.check(got[q], FR.exact(a[q], b[q]), D)


def test_feature_distance_at_scale():
    """1024 x 1024 x 512 x 8 sequences: every output finite and within the bound of float64 cdist, and 64 sampled rows of every
    sequence within the derived bound of extended precision"""
    rng = np.random.default_rng(3)
    a = (rng.normal(0, 1, (8, 1024, 512)) / 22.6).astype(np.float32)
    b = (rng.normal(0, 1, (8, 1024, 512)) / 22.6).astype(np.float32)
    b[:, :16] = a[:, :16]
    got = _dist(a, b)
    assert np.isfinite(got).all() and (got >= 0).all()
    assert (np.diagonal(got[:, :16, :16], axis1=1, axis2=2) == 0).all()
    # every output against float64 cdist, whose own error has the same bound: |got - cdist| <= 2 gamma_{D+3} cdist
    from scipy.spatial.distance import cdist
    for q in range(8):
        ref = cdist(a[q].astype(np.float64), b[q].astype(np.float64))
        assert (np.abs(got[q] - ref) <= 2 * FR.gamma(512 + 3) * (1 + 1e-9) * ref).all(), "sequence %d" % q
    for q in range(8):
        rows = rng.choice(1024, 64, replace=False)
        FR.check(got[q][rows], FR.exact(a[q][rows], b[q]), 512, "sequence %d" % q)
