"""not-gpu: the oracle's trackers against the reference's track life cycle (tests/golden/loop_lifecycle.npz): births and deaths
mid-stream, long occlusions that outlive max_time_lost, duplicate tracks, empty frames, scores exactly on the thresholds,
non-default options and every Kalman format with every tracker kind."""
import numpy as np
import pytest

import lifecycle_golden as LG
from oracle import kalman as K, refshim, trackers as T

CONFIGS = LG.configs()


def run_oracle(cfg):
    frames, warps = cfg.stream()
    orc = T.TrackerOracle(**cfg.oracle_kwargs())
    for i, f in enumerate(frames):
        out = orc.update(f, None if warps is None else warps[i])
        yield i, orc, out


@pytest.mark.parametrize("name", CONFIGS)
def test_oracle_lifecycle_matches_reference(name):
    cfg = LG.Config(name)
    for i, orc, out in run_oracle(cfg):
        where = "%s frame %d" % (name, i + 1)
        assert [o[0] for o in out] == cfg.out_ids[i].tolist(), where
        assert np.array_equal(np.array([o[2] for o in out], np.float32), cfg.out_cls[i]), where
        assert orc.removed_now_ids == cfg.rem_ids[i].tolist(), where
        for which in ("tracked", "lost"):
            rows, tlwh = orc.list_rows(which)
            assert np.array_equal(rows, cfg.rows[which][i]), "%s: %s list" % (where, which)
            if i in cfg.tlwh_frames:
                assert np.array_equal(tlwh, cfg.tlwh[(which, i)]), "%s: %s boxes" % (where, which)
        if i in cfg.tlwh_frames:
            assert np.array_equal(np.array([o[1] for o in out]).reshape(-1, 4), cfg.tlwh[("out", i)]), where


@pytest.mark.parametrize("name", CONFIGS)
def test_lifecycle_golden_exercises_the_state_machine(name):
    """Coverage floors: a change of the stream generator or of the configurations cannot quietly stop exercising pruning,
    late re-activation, duplicate removal, empty frames, threshold ties or births."""
    cfg = LG.Config(name)
    e = cfg.events
    assert e["prunes"] >= 10, e
    assert e["duplicate_drops"] >= 5, e
    assert e["empty_frames"] >= 3, e
    assert e["threshold_ties"] >= 100, e
    assert e["births"] >= 60, e
    if cfg.max_time_lost >= 20:
        assert e["reactivated_after_10"] >= 10, e
    # the stored lists agree with the counted events (a duplicate dropped in the frame it was born never shows in the lists)
    prunes, dups = cfg.events_until(cfg.n_frames)
    assert prunes == e["prunes"] and 0 < dups <= e["duplicate_drops"], (prunes, dups, e)


def test_nsa_kalman_paths_match_reference():
    """NSAKalmanFilter with a float32 confidence: projection and update from the float32 mean STrack.activate leaves (the
    first update of every new track under kalman_format='strongsort'), and from a float64 mean.  The float32 path squares the
    (1 - conf)-scaled noise in float32, as NumPy does for an all-float32 list."""
    g = LG.load()
    fmt = K.FMT_NSA
    n = len(g["nsa_z0"])
    m0, c0 = zip(*[K.initiate(fmt, z) for z in g["nsa_z0"]])
    assert np.array_equal(np.stack(m0), g["nsa_init_mean"]) and np.array_equal(np.stack(c0), g["nsa_init_cov"])
    c0_, c1, c2 = g["nsa_conf0"], g["nsa_conf1"], g["nsa_conf2"]
    pm, ps = zip(*[K.project(fmt, m0[i], c0[i], mean_f32=True, confidence=c0_[i]) for i in range(n)])
    assert np.array_equal(np.stack(pm), g["nsa_proj32_mean"]) and np.array_equal(np.stack(ps), g["nsa_proj32_cov"])
    um, uc = zip(*[K.update(fmt, m0[i], c0[i], g["nsa_z1"][i], mean_f32=True, confidence=c0_[i]) for i in range(n)])
    assert np.array_equal(np.stack(um), g["nsa_upd32_mean"]) and np.array_equal(np.stack(uc), g["nsa_upd32_cov"])
    mp, cp = K.multi_predict(fmt, np.stack(um), np.stack(uc))
    assert np.array_equal(mp, g["nsa_pred_mean"]) and np.array_equal(cp, g["nsa_pred_cov"])
    pm, ps = zip(*[K.project(fmt, mp[i], cp[i], confidence=c1[i]) for i in range(n)])
    assert np.array_equal(np.stack(pm), g["nsa_proj64_mean"]) and np.array_equal(np.stack(ps), g["nsa_proj64_cov"])
    um, uc = zip(*[K.update(fmt, mp[i], cp[i], g["nsa_z2"][i], confidence=c2[i]) for i in range(n)])
    assert np.array_equal(np.stack(um), g["nsa_upd64_mean"]) and np.array_equal(np.stack(uc), g["nsa_upd64_cov"])


@pytest.mark.skipif(not refshim.available(), reason="the reference tree is not present")
@pytest.mark.parametrize("name", ["bytetrack_strongsort", "botsort_c01_tb10"])
def test_golden_generator_reproduces_fixture(name):
    """The fixture generator, run on the reference here, writes what is committed (the stream and the reference are deterministic)."""
    import importlib.util
    import os
    spec = importlib.util.spec_from_file_location("make_golden_lifecycle", os.path.join(os.path.dirname(LG.PATH), "make_golden_lifecycle.py"))
    gen = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(gen)
    i = [c[0] for c in gen.CONFIGS].index(name)
    fresh = gen.run_config(refshim.load(), *gen.CONFIGS[i], seed=300 + i)
    g = LG.load()
    for k, v in fresh.items():
        assert np.array_equal(np.asarray(v), g[k]), k
