"""gpu: UAVMOT on the H100 (TrackEngine("uavmot"), B2T_UAVMOT).
  * the reference's goldens (tests/golden/loop_uavmot.npz): ids exact, tlwh within 1e-9, lists exact;
  * four different sequences in one launch give bitwise the results of each sequence alone;
  * a 300-object stream against the oracle (tests/uavmot_oracle.py): ids exact;
  * b2t_structure_vectors / b2t_structure_distance against the oracle at their edges: empty sets, one point, coincident points, ties,
    400, diagonals, and a 1000-point set."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu
torch = pytest.importorskip("torch")

from b200track.synth import make_stream          # noqa: E402
import uavmot_golden as UG                       # noqa: E402
import uavmot_oracle as U                        # noqa: E402


def _engine(n_seq=1, dtype="f64", cap=256, dmax=128, **kw):
    from b200track.engine import TrackEngine
    return TrackEngine("uavmot", n_seq=n_seq, dtype=dtype, cap=cap, dmax=dmax, **kw)


def _int_rows(rows):
    return rows[:, [0, 8, 9, 11, 12, 10]].astype(np.int64)


@pytest.mark.parametrize("name", [c.name for c in UG.CONFIGS])
def test_engine_matches_reference(name):
    cfg = next(c for c in UG.CONFIGS if c.name == name).load()
    eng = _engine(kalman_format=cfg.fmt, track_buffer=cfg.track_buffer)
    for i, fr in enumerate(cfg.stream()):
        where = "%s frame %d" % (name, i + 1)
        res = eng.step([fr])[0]
        assert res[:, 0].astype(np.int64).tolist() == cfg.ids[i].tolist(), where
        np.testing.assert_allclose(res[:, 1:5], cfg.tlwh[i], rtol=0, atol=1e-9, err_msg=where)
        for which in ("tracked", "lost"):
            assert np.array_equal(_int_rows(eng.read_list(0, which)), cfg.lists[which][i]), "%s: %s list" % (where, which)


def test_four_sequences_in_one_launch_equal_each_alone():
    streams = [UG.make_uavmot_stream(200 + q, 40) for q in range(3)] + [make_stream(7, 40, n_obj=120)[0]]
    many = _engine(n_seq=4, cap=512, dmax=256)
    ones = [_engine(cap=512, dmax=256) for _ in range(4)]
    for i in range(40):
        got = [r.copy() for r in many.step([s[i] for s in streams])]
        for q in range(4):
            alone = ones[q].step([streams[q][i]])[0]
            assert np.array_equal(got[q], alone), "frame %d sequence %d" % (i + 1, q)


def test_300_objects_match_oracle():
    frames, _ = make_stream(31, 40, n_obj=300)
    eng = _engine(cap=1024, dmax=512)
    orc = U.UavmotOracle()
    for i, fr in enumerate(frames):
        res = eng.step([fr])[0]
        exp = orc.update(fr)
        assert res[:, 0].astype(int).tolist() == [t[0] for t in exp], "frame %d" % (i + 1)


def _sets():
    rng = np.random.default_rng(4)
    lat = rng.integers(0, 9, (60, 2)).astype(np.float64) * 100
    return [np.zeros((0, 2)), np.array([[1.5, 2.5]]), np.full((9, 2), 640.0), np.array([[0, 0], [400, 0], [0, 399.5], [250, 250]]),
            lat, lat + rng.integers(-1, 2, lat.shape), rng.uniform(0, 1280, (1000, 2))]


def test_structure_entries_match_oracle():
    from b200track.engine import ops
    o = ops()
    for pts in _sets():
        for det in (False, True):
            p = pts.astype(np.float32 if det else np.float64)
            got = o.structure_vectors(o.dev(p.reshape(-1, 2), torch.float32 if det else torch.float64), detection=det).cpu().numpy()
            assert np.array_equal(got, U.structure_vectors(p, det)), "n=%d detection=%s" % (len(p), det)
        a, b = U.structure_vectors(pts), U.structure_vectors(pts.astype(np.float32), True)
        if len(a):
            got = o.structure_distance(o.dev(a, torch.float64), o.dev(b, torch.float64)).cpu().numpy()
            assert np.array_equal(got, U.structure_distance(a, b)), "n=%d" % len(a)
