"""not-gpu: the StrongSORT oracle (tests/strongsort_oracle.py) reproduces the unmodified reference's goldens
(tests/golden/loop_strongsort.npz) bit for bit: ids, tlwh, the tracked and lost lists with their states, and the features."""
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import strongsort_golden as SG                       # noqa: E402
from strongsort_oracle import StrongSortOracle       # noqa: E402


@pytest.mark.parametrize("name", [c.name for c in SG.CONFIGS])
def test_oracle_matches_reference(name):
    cfg = next(c for c in SG.CONFIGS if c.name == name).load()
    frames, feats, warps = cfg.stream()
    orc = StrongSortOracle(gamma=cfg.gamma, use_ecc=cfg.use_ecc, kalman_format=cfg.fmt, track_buffer=cfg.track_buffer)
    for i in range(cfg.n_frames):
        where = "%s frame %d" % (name, i + 1)
        res = orc.update(frames[i], feats[i], warps[i] if cfg.use_ecc else None)
        assert [t[0] for t in res] == cfg.ids[i].tolist(), where
        assert np.array_equal(np.array([t[1] for t in res]).reshape(-1, 4), cfg.tlwh[i]), where
        for which in ("tracked", "lost"):
            rows, _ = orc.list_rows(which)
            assert np.array_equal(rows, cfg.lists[which][i]), "%s: %s list" % (where, which)
        if i in cfg.feats:
            assert np.array_equal(orc.last_features().reshape(len(res), -1), cfg.feats[i]), where
