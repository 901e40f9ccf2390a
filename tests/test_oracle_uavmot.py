"""not-gpu: the UAVMOT oracle (tests/uavmot_oracle.py) reproduces the reference's goldens (tests/golden/loop_uavmot.npz) bit for bit,
and its structure vectors and distances equal the reference's matching.structure_representation / cdist where the reference tree is
present."""
import numpy as np
import pytest

import uavmot_golden as UG
import uavmot_oracle as U
from oracle import refshim


@pytest.mark.parametrize("name", [c.name for c in UG.CONFIGS])
def test_oracle_matches_golden(name):
    cfg = next(c for c in UG.CONFIGS if c.name == name).load()
    orc = U.UavmotOracle(kalman_format=cfg.fmt, track_buffer=cfg.track_buffer)
    for i, fr in enumerate(cfg.stream()):
        res = orc.update(fr)
        assert [t[0] for t in res] == cfg.ids[i].tolist(), "frame %d" % (i + 1)
        assert np.array_equal(np.array([t[1] for t in res]).reshape(-1, 4), cfg.tlwh[i]), "frame %d" % (i + 1)
        for w in ("tracked", "lost"):
            assert np.array_equal(orc.list_rows(w)[0], cfg.lists[w][i]), "frame %d: %s list" % (i + 1, w)


class _Pt:
    def __init__(self, mean=None, xy=None):
        self.mean, self._xy = mean, xy

    def get_xy(self):
        return self._xy


def point_sets():
    rng = np.random.default_rng(3)
    sets = [np.zeros((0, 2)), np.array([[5.0, 5.0]]), np.full((6, 2), 7.0), np.array([[0, 0], [400, 0], [0, 399], [300, 300]], float)]
    for k in range(12):
        n = int(rng.integers(2, 40))
        sets.append(rng.uniform(0, 900, (n, 2)) if k % 2 else rng.integers(0, 9, (n, 2)).astype(np.float64) * 100)
    return sets


@pytest.mark.skipif(not refshim.available(), reason="needs the reference tree")
def test_structure_matches_reference():
    from scipy.spatial.distance import cdist
    ref = refshim.load()
    for pts in point_sets():
        if len(pts) == 0:
            continue
        a = ref.matching.structure_representation([_Pt(mean=np.r_[p, np.zeros(6)]) for p in pts])
        assert np.array_equal(a, U.structure_vectors(pts))
        d32 = pts.astype(np.float32)
        b = ref.matching.structure_representation([_Pt(xy=p) for p in d32], mode="detection")
        assert np.array_equal(b, U.structure_vectors(d32, True))
        assert np.array_equal(np.maximum(0.0, cdist(a, b, "cosine")), U.structure_distance(a, b))
