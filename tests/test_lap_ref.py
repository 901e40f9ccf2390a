"""not-gpu: pins tests/lap_ref.py -- the rectangular scipy solver, its uniqueness certificate and the CSR layouts -- against
oracle/lapjv.py's square extension and against brute force, on the CPU."""
import math

import numpy as np
import pytest

import lap_ref as R
from oracle import lapjv as olap


def test_solve_matches_square_extension_and_brute_force():
    rng = np.random.default_rng(0)
    for _ in range(150):
        n, m = int(rng.integers(0, 5)), int(rng.integers(0, 5))
        t = float(rng.choice([0.5, 0.9, 3.0]))
        cost = rng.uniform(-2, 1.5, (n, m))
        cost[rng.uniform(size=(n, m)) < 0.2] = np.inf
        obj, x = R.solve(cost, t)
        if n and m:
            best, bx, uniq = olap.brute_force(np.where(np.isfinite(cost), cost, 1e9), t)
            assert obj == pytest.approx(best, abs=1e-12)
            fin = np.where(np.isfinite(cost), cost, 1e9)
            o2, x2, _ = olap.lapjv(fin, True, t)
            assert obj == pytest.approx(olap.objective(fin, x2, t), abs=1e-12)
            if uniq:
                assert np.array_equal(x, bx)
        R.check_matching(cost, t, x, R.y_of(x, m))


def test_nan_inf_and_threshold_are_not_eligible():
    t = 0.7
    cost = np.array([[np.nan, np.inf, t, -np.inf]])
    assert not R.eligible(cost, t)[0, :3].any() and R.eligible(cost, t)[0, 3]


def test_certificate_gap():
    # optimum {(0,1), (1,0)} = -2.0; dropping either edge leaves at best one edge, weight 1.5 - 0.5 ... the gap is exact here
    t = 0.5
    cost = t - np.array([[0.2, 1.0], [1.0, 0.3]])
    obj, x, gap = R.certify(cost, t)
    assert list(x) == [1, 0] and obj == -2.0 and gap == pytest.approx(2.0 - 1.0)
    tied = np.full((2, 2), 0.1)
    assert R.certify(tied, t)[2] == 0.0
    assert R.certify(np.full((2, 2), 1.0), t)[2] == math.inf        # nothing eligible


def test_counterexamples_have_the_stated_optima():
    a = 0.9 - np.array([[1001.00001, 1.0], [1000.00003, -0.05]])
    obj, x, gap = R.certify(a, 0.9)
    assert list(x) == [1, 0] and obj == pytest.approx(-1001.00003, abs=1e-9) and gap > 1e-6
    b = 0.5 - np.array([[1000.00002], [1000.00003]])
    obj, x, gap = R.certify(b, 0.5)
    assert list(x) == [-1, 0] and gap > 5e-6


def test_csr_layout_and_poison():
    rng = np.random.default_rng(1)
    cost = rng.uniform(0, 1.2, (12, 9))
    t = 0.9
    rows = R.rows_of(cost, t, rng, pad=0.5, shuffle=True)
    for name, (s_cap, w2) in R.placements(rows).items():
        c = R.Csr(12, 9, t, rows, s_cap, w2, seed=3)
        assert c.n_entries == sum(len(r) for r in rows)
        end = c.row_start + c.row_cnt
        for e in range(c.n_entries):
            i = c.owner[e]
            assert c.row_start[i] <= e < end[i]
            shared = end[i] <= s_cap
            if shared:          # shared rows are read from the mirror, never from the global copy
                assert c.m_col[e] == c.col[e] and c.m_cost[e] == c.cost[e]
                if c.col[e] >= 0:
                    assert c.e_cost[e] == t - 1e6
            elif w2[0] <= e < w2[1]:
                assert c.m_col[e] == c.col[e] and c.m_row[e] == i
            else:
                assert c.e_col[e] == c.col[e] and c.e_row[e] == i and c.m_cost[e] == t - 1e6
        assert np.array_equal(np.where(np.isfinite(c.dense()), c.dense(), 5.0)[R.eligible(cost, t)], cost[R.eligible(cost, t)])
    assert {"s_mid_row", "s_at_row_end", "w2_straddle_end", "all_shared", "global"} <= set(R.placements(rows))


def test_f32_bound_is_positive_and_cubic():
    c = np.random.default_rng(2).uniform(0, 1, (10, 10))
    b10 = R.f32_shortfall_bound(c, 0.9)
    b20 = R.f32_shortfall_bound(np.tile(c, (2, 2)), 0.9)
    assert 0 < b10 < 1e-2 and b20 > 4 * b10
