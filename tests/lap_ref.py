"""Exact reference for the thresholded assignment solver (csrc/b2t_lap.cuh), and the CSR layouts the fused step hands it.

TEST INFRASTRUCTURE.  The solver promises the optimum of ``lap.lapjv(cost, extend_cost=True, cost_limit=t)``, i.e.

    minimise  sum over matched (i, j) of (c_ij - t)   over partial matchings using only pairs with c_ij < t.

``solve`` finds it with ``scipy.optimize.linear_sum_assignment`` on the RECTANGULAR formulation -- an n x (m + n) matrix with
c_ij - t on the eligible pairs, one private 0-cost dummy column per row ("stay unmatched") and +inf everywhere else -- which is
independent of the square (n + m)^2 extension ``oracle/lapjv.py`` restates (tests/test_lap_ref.py pins the two against each other
and against ``brute_force``).  Objectives are summed with ``math.fsum`` from the float64 costs, so they are exact up to one final
rounding.

``certify`` proves the optimum unique with a gap: it forbids each matched edge in turn and re-solves.  Any other matching either
lacks some edge of the optimum (so it is no better than that re-solve) or strictly contains the optimum (impossible: the extra
edge has positive weight t - c, so the optimum would not be optimal).  So every other matching is worse by at least
``gap = min over matched edges (re-solve - optimum)``; indices are compared only when the gap is certified.

Float32.  Float32 costs and thresholds are exact in float64, so the float64 optimum of the float32 problem is the reference, and
``f32_shortfall_bound`` says how far the float32 solver's objective may fall short of it (derivation at the function).
"""
import math

import numpy as np
from scipy.optimize import linear_sum_assignment

U32 = 2.0 ** -24        # unit roundoff of float32


def eligible(cost, t):
    """The pairs the reference may match: c < t (NaN and +inf fail the comparison, as in lap's and the kernel's c < t)."""
    with np.errstate(invalid="ignore"):
        return np.asarray(cost, np.float64) < t


def objective(cost, x, t):
    """sum over matched rows of (c_ij - t), exactly summed (math.fsum of the float64 terms c and -t)."""
    cost = np.asarray(cost, np.float64)
    terms = []
    for i, j in enumerate(np.asarray(x)):
        if j >= 0:
            terms += [float(cost[i, j]), -float(t)]
    return math.fsum(terms)


def solve(cost, t, forbid=None):
    """Exact optimum (objective, x) of the thresholded problem; forbid: an (i, j) pair to exclude."""
    cost = np.asarray(cost, np.float64)
    n, m = cost.shape
    if n == 0:
        return 0.0, np.zeros(0, np.int64)
    ok = eligible(cost, t)
    if forbid is not None:
        ok = ok.copy()
        ok[forbid] = False
    a = np.full((n, m + n), np.inf)
    a[:, :m] = np.where(ok, cost - t, np.inf)
    a[np.arange(n), m + np.arange(n)] = 0.0
    r, c = linear_sum_assignment(a)
    x = np.full(n, -1, np.int64)
    x[r] = np.where(c < m, c, -1)
    return objective(cost, x, t), x


def certify(cost, t, x=None, obj=None):
    """Returns (obj, x, gap): the optimum and the certified margin by which every other matching is worse (inf when the optimum
    is empty, i.e. nothing is eligible)."""
    if x is None:
        obj, x = solve(cost, t)
    gap = math.inf
    for i, j in enumerate(x):
        if j >= 0:
            o2, _ = solve(cost, t, forbid=(i, int(j)))
            gap = min(gap, o2 - obj)
    return obj, x, gap


def y_of(x, m):
    y = np.full(m, -1, np.int64)
    for i, j in enumerate(x):
        if j >= 0:
            y[j] = i
    return y


def check_matching(cost, t, x, y):
    """x / y are a valid matching of eligible pairs, consistent with each other."""
    cost = np.asarray(cost, np.float64)
    n, m = cost.shape
    ok = eligible(cost, t)
    assert len(x) == n and len(y) == m
    for i, j in enumerate(x):
        if j >= 0:
            assert j < m and ok[i, j], "row %d matched to ineligible column %d" % (i, j)
    assert np.array_equal(np.asarray(y), y_of(x, m)), "x and y disagree"


# ---------------------------------------------------------------------------------------------------------------- float32
def f32_shortfall_bound(cost, t):
    """How far the float32 solver's objective (evaluated exactly) may exceed the optimum.

    The solver (lap_augment_row) keeps duals u_i (rows), v_j (columns) in float32 and works on c'_ij = c_ij - t/2, with each row's
    dummy at cost t/2 (t/2 is exact).  An exact run keeps, for every live edge, r_ij = c'_ij - u_i - v_j >= 0, r = 0 on matched
    edges, t/2 - u_i >= 0 with equality for a row left on its dummy, and v_j <= 0 (v only decreases: v -= minval - dist, with
    dist <= minval for a scanned column) with v_j = 0 on never-scanned (so unmatched) columns.  Summing over the returned matching
    M and any other matching M' then gives cost(M) = sum u + sum v <= cost(M').  With rounding each of those relations holds up
    to an error e, and the same sums give

        cost(M) - cost(M')  <=  2 * n * e        (n rows: one relation per row for M, one per row for M').

    e collects, for one edge, (a) the rounding of the reduced cost minval + ((c - t/2) - u) - v that decided the search -- four
    float32 operations on operands bounded by D, at most 4 * U32 * 2D each time it is evaluated -- and (b) the drift of u_i and v_j
    from their exact values: each of the n augmentations updates each dual at most once (u += d, v -= d), one rounding of at most
    U32 * 2D each, so at most 2 * n * U32 * 2D for the pair.  D bounds every magnitude the search handles: each dual and each
    distance is a sum of at most 2n reduced costs along an alternating path, each at most C = max |c' | + t/2 over the eligible
    pairs, so D = 2 n C + C.  Altogether

        e <= (4 + 2 n) * U32 * 2 D,     shortfall <= 2 n e.

    This is a first-order bound (products of two rounding errors are dropped) and it is cubic in n: at unit-sized weights it is
    ~1e-4 for 4 rows, ~0.1 for 40 and ~200 for 512, so it decides index equality only for small problems and says nothing about the
    large float32 cases -- those are held to the objective within it and, on tie-free generators, to the reference's indices.
    Kernelisation adds nothing: its rule fires only on edges that belong to every optimum (b2t_lap.cuh, lap_kernelize_rows)."""
    cost = np.asarray(cost, np.float64)
    n = cost.shape[0]
    ok = eligible(cost, t)
    if n == 0 or not ok.any():
        return 0.0
    C = float(np.max(np.abs(cost[ok] - t / 2.0))) + abs(t) / 2.0
    D = (2 * n + 1) * C
    e = (4 + 2 * n) * U32 * 2 * D
    return 2 * n * e


# ---------------------------------------------------------------------------------------------------------------- CSR layouts
class Csr:
    """One problem laid out as build_csr / build_csr_dense lay it out: rows contiguous and in order, each row's entries
    (col, cost) with col -1 for padding, plus the storage placement.

    Every entry has ONE authoritative copy the solver may read: the shared-memory mirror (m_*) for a row ending at or below s_cap,
    the global arrays (e_*) for the other rows, and additionally the second window (also m_*) for entries inside
    [w2_base, w2_end).  Every other copy is POISON -- a live-looking column with a very attractive cost -- so that a storage path
    reading the wrong copy changes the result instead of reading an identical value.  (One exception, forced by the single mirror
    array feeding both windows: a window entry below s_cap keeps its true value in the shared copy too.)"""

    def __init__(self, n, m, t, rows, s_cap=0, w2=(0, 0), rowwise=False, seed=0, poison=True):
        self.n, self.m, self.t = n, m, float(t)
        self.rows = rows                               # list of lists of (col, cost)
        self.row_cnt = np.array([len(r) for r in rows], np.int32)
        self.row_start = np.zeros(n, np.int32)
        if n:
            self.row_start[1:] = np.cumsum(self.row_cnt)[:-1]
        self.n_entries = int(self.row_cnt.sum())
        self.s_cap, self.w2, self.rowwise = int(s_cap), (int(w2[0]), int(w2[1])), bool(rowwise)
        ne = self.n_entries
        col = np.full(ne, -1, np.int32)
        cst = np.zeros(ne, np.float64)
        own = np.full(ne, -1, np.int32)
        for i, r in enumerate(rows):
            for k, (j, c) in enumerate(r):
                e = self.row_start[i] + k
                col[e], cst[e], own[e] = j, c, i
        self.col, self.cost, self.owner = col, cst, own
        end = self.row_start + self.row_cnt
        shared = np.zeros(ne, bool)
        in_win = np.zeros(ne, bool)
        row_in_win = np.zeros(ne, bool)
        b, w = self.w2
        for e in range(ne):
            i = own[e]
            shared[e] = end[i] <= self.s_cap
            in_win[e] = b <= e < w
            row_in_win[e] = self.row_start[i] >= b and end[i] <= w
        rng = np.random.default_rng(seed)
        pc = rng.integers(0, max(m, 1), ne).astype(np.int32)
        pw = np.full(ne, self.t - 1e6)                 # weight 1e6: any read of it changes the optimum
        pr = rng.integers(0, max(n, 1), ne).astype(np.int32)
        # global copy: poisoned where shared memory or the window holds the row entirely
        g_bad = (shared | (row_in_win & ~shared)) if poison else np.zeros(ne, bool)
        self.e_col = np.where(g_bad, pc, col).astype(np.int32)
        self.e_cost = np.where(g_bad, pw, cst)
        self.e_row = np.where(g_bad, pr, own).astype(np.int32)
        # mirror: true for shared rows and inside the window; the buffer's tail past w2_end is poison too
        m_good = shared | in_win
        m_bad = ~m_good if poison else np.zeros(ne, bool)
        self.m_col = np.where(m_bad, pc, col).astype(np.int32)
        self.m_cost = np.where(m_bad, pw, cst)
        self.m_row = np.where(m_bad, pr, own).astype(np.int32)

    def dense(self):
        """The problem as a dense matrix (+inf = not listed)."""
        c = np.full((self.n, self.m), np.inf)
        for i, r in enumerate(self.rows):
            for j, v in r:
                if j >= 0:
                    c[i, j] = v
        return c


def rows_of(cost, t, rng=None, pad=0.0, shuffle=False):
    """CSR rows of a dense problem: the eligible pairs (c < t), optionally shuffled within a row and with col -1 padding entries
    inserted (pad = padding entries per real entry, on average)."""
    cost = np.asarray(cost, np.float64)
    ok = eligible(cost, t)
    rows = []
    for i in range(cost.shape[0]):
        r = [(int(j), float(cost[i, j])) for j in np.nonzero(ok[i])[0]]
        if shuffle and rng is not None:
            rng.shuffle(r)
        if pad and rng is not None:
            for _ in range(int(rng.poisson(pad * max(len(r), 1)))):
                r.insert(int(rng.integers(0, len(r) + 1)), (-1, float(t) - 7.0))
        rows.append(r)
    return rows


def placements(csr_rows):
    """Named (s_cap, (w2_base, w2_end)) placements for a row list: mid-row, exactly at a row end, a row straddling w2_end,
    s_cap = 0, and everything in shared memory."""
    cnt = [len(r) for r in csr_rows]
    start = np.concatenate([[0], np.cumsum(cnt)]).astype(int)
    ne = int(start[-1])
    long_rows = [i for i in range(len(cnt)) if cnt[i] >= 3]
    out = {"global": (0, (0, 0)), "all_shared": (ne, (0, 0))}
    if long_rows:
        a = long_rows[len(long_rows) // 3]
        b = long_rows[(2 * len(long_rows)) // 3]
        mid_a = int(start[a] + cnt[a] // 2)
        mid_b = int(start[b] + cnt[b] // 2)
        out["s_mid_row"] = (mid_a, (0, 0))
        out["s_at_row_end"] = (int(start[a + 1]), (0, 0))
        # the step's window starts at the first spilled row -- which straddles s_cap -- and may end inside a row
        out["w2_from_straddler"] = (mid_a, (int(start[a]), mid_b if mid_b > start[a] else ne))
        out["w2_straddle_end"] = (0, (int(start[a]), mid_b if mid_b > start[a] else ne))
        out["w2_at_row_end"] = (int(start[a]), (int(start[a]), int(start[b + 1])))
        out["w2_to_end"] = (0, (mid_a, ne))
    return out
