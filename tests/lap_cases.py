"""The assignment solver's cases, shared by the simulator tier (tests/test_hostsim_lap.py, reduced sizes) and the H100 tier
(tests/test_gpu_lap.py, full sizes).  Each case names the solver path it targets and asserts, through the counters
b2t_lap_solve_csr returns, that it reached it; every result is checked against the exact reference of tests/lap_ref.py.

A backend moves arrays to and from the library's memory: ``dev(np_array) -> handle``, ``ptr(handle)``, ``host(handle)``."""
import ctypes as C
import math

import numpy as np

import lap_ref as R
from b200track import _lib as L

CERTIFY_MAX_ROWS = 300          # certify uniqueness up to this many rows; above, compare with the reference on tie-free generators
F64_U = 2.0 ** -53


def npdt(dtype):
    return np.float64 if dtype == L.F64 else np.float32


def as_dtype(cost, t, dtype):
    """The problem the solver sees: costs and threshold rounded to the dtype (exact in float64)."""
    return np.asarray(cost, npdt(dtype)).astype(np.float64), float(npdt(dtype)(t))


class Report(dict):
    def line(self):
        return " ".join("%s=%s" % kv for kv in sorted(self.items()))


def check(cost, t, dtype, x, y, report, certify=True, ref=None):
    """x / y: a valid matching whose objective is within the dtype's shortfall bound of the optimum; indices equal to the
    optimum's wherever the certified gap exceeds that bound."""
    cost, t = as_dtype(cost, t, dtype)
    n, m = cost.shape
    R.check_matching(cost, t, x, y)
    obj = R.objective(cost, x, t)
    if ref is None:
        if certify and n <= CERTIFY_MAX_ROWS:
            ref = R.certify(cost, t)
        else:
            o, xr = R.solve(cost, t)
            ref = (o, xr, None)
    opt, xr, gap = ref
    bound = R.f32_shortfall_bound(cost, t) if dtype == L.F32 else R.f32_shortfall_bound(cost, t) * F64_U / R.U32
    short = obj - opt
    assert short <= bound, "objective %r falls short of the optimum %r by %r > bound %r" % (obj, opt, short, bound)
    if gap is None:                 # large tie-free generator, gaps far above the rounding of either dtype: the reference's indices
        assert np.array_equal(np.asarray(x), xr), "assignment differs from the reference (uncertified, tie-free generator)"
    elif gap > bound:
        assert np.array_equal(np.asarray(x), xr), "assignment differs from the certified unique optimum (gap %r)" % gap
    report["gap"] = min(report.get("gap", math.inf), gap if gap is not None else math.inf)
    if dtype == L.F32 and bound > 0:
        report["f32_short/bound"] = max(report.get("f32_short/bound", 0.0), short / bound)
    return obj, opt


# ---------------------------------------------------------------------------------------------------------------- entries
def solve_csr(be, dtype, csrs, expect_rc=0, mirrors=True, row_index=True):
    """All problems of `csrs` (lap_ref.Csr) in ONE launch of b2t_lap_solve_csr.  Returns [(x, y, counters)] per problem.
    mirrors=False passes m_* = NULL (the mirrors are copies of e_*), row_index=False passes e_row = m_row = NULL."""
    lib = be.lib
    probs = (L.LapCsrProblem * len(csrs))()
    rs, rc, ec, ew, er, mc, mw, mr = [], [], [], [], [], [], [], []
    ro = co = eo = 0
    for k, c in enumerate(csrs):
        probs[k] = L.LapCsrProblem(n=c.n, m=c.m, thresh=c.t, row_off=ro, col_off=co, entry_off=eo, n_entries=c.n_entries,
                                   s_cap=c.s_cap, w2_base=c.w2[0], w2_end=c.w2[1], rowwise=int(c.rowwise))
        rs.append(c.row_start); rc.append(c.row_cnt)
        ec.append(c.e_col); ew.append(c.e_cost); er.append(c.e_row); mc.append(c.m_col); mw.append(c.m_cost); mr.append(c.m_row)
        ro += c.n; co += c.m; eo += c.n_entries
    cat = lambda a, dt: np.ascontiguousarray(np.concatenate(a + [np.zeros(1, dt)]).astype(dt))      # never empty
    dt = npdt(dtype)
    arrs = [be.dev(cat(rs, np.int32)), be.dev(cat(rc, np.int32)), be.dev(cat(ec, np.int32)), be.dev(cat(ew, dt)),
            be.dev(cat(er, np.int32)), be.dev(cat(mc, np.int32)), be.dev(cat(mw, dt)), be.dev(cat(mr, np.int32))]
    x = be.dev(np.full(ro + 1, -9, np.int32)); y = be.dev(np.full(co + 1, -9, np.int32))
    cnt = be.dev(np.full(len(csrs) * L.LAP_COUNTERS, -9, np.int32))
    ws = be.dev(np.zeros(lib.b2t_lap_csr_workspace_bytes(len(csrs)), np.uint8))
    launches = lib.b2t_launch_count()
    ptrs = [be.ptr(a) for a in arrs]
    if not row_index:
        ptrs[4] = ptrs[7] = None
    if not mirrors:
        ptrs[5] = ptrs[6] = ptrs[7] = None
    rcode = lib.b2t_lap_solve_csr(dtype, C.cast(probs, C.c_void_p), len(csrs), *ptrs, be.ptr(x), be.ptr(y), be.ptr(cnt),
                                  be.ptr(ws), lib.b2t_lap_csr_workspace_bytes(len(csrs)), None)
    if expect_rc:
        assert rcode == expect_rc, "expected return code %d, got %d" % (expect_rc, rcode)
        assert lib.b2t_launch_count() == launches, "launched although the problem does not fit"
        return None
    L.check(lib, rcode)
    be.sync()
    xh, yh, ch = be.host(x), be.host(y), be.host(cnt).reshape(len(csrs), L.LAP_COUNTERS)
    out, ro, co = [], 0, 0
    for k, c in enumerate(csrs):
        out.append((xh[ro:ro + c.n].astype(np.int64), yh[co:co + c.m].astype(np.int64), ch[k].copy()))
        ro += c.n; co += c.m
    return out


def solve_dense(be, dtype, cost, t, expect_rc=0):
    lib = be.lib
    cost = np.asarray(cost)
    n, m = cost.shape
    c = be.dev(np.ascontiguousarray(cost, npdt(dtype)) if cost.size else np.zeros(1, npdt(dtype)))
    x = be.dev(np.full(max(n, 1), -9, np.int32)); y = be.dev(np.full(max(m, 1), -9, np.int32))
    wsb = lib.b2t_lap_workspace_bytes(dtype, n, m, 1)
    ws = be.dev(np.zeros(wsb, np.uint8))
    launches = lib.b2t_launch_count()
    rcode = lib.b2t_lap_solve(dtype, be.ptr(c), n, m, max(m, 1), float(t), be.ptr(x), be.ptr(y), be.ptr(ws), wsb, 1, None)
    if expect_rc:
        assert rcode == expect_rc, "expected return code %d, got %d" % (expect_rc, rcode)
        assert lib.b2t_launch_count() == launches, "launched although the problem does not fit"
        return None
    L.check(lib, rcode)
    be.sync()
    return be.host(x)[:n].astype(np.int64), be.host(y)[:m].astype(np.int64)


def run_one(be, dtype, cost, t, rows=None, rowwise=False, **kw):
    """One problem through b2t_lap_solve_csr, everything in global memory."""
    cost = np.asarray(cost, np.float64)
    n, m = cost.shape
    c32, t32 = as_dtype(cost, t, dtype)
    rows = R.rows_of(c32, t32) if rows is None else rows
    return solve_csr(be, dtype, [R.Csr(n, m, t32, rows, rowwise=rowwise, poison=False, **kw)])[0]


def lap_smem_bytes(n, m, tsize, csr=False, s_cap=0, w2=0):
    """Shared memory of lap_solve_kernel (csr=False) / lap_solve_csr_kernel: the Arena takes of LapWork::size, then the CSR
    entry's mirror and window takes (an empty take still takes one element), + 16."""
    off = 0

    def take(sz, k):
        nonlocal off
        off = (off + 15) & ~15
        off += sz * max(k, 1)
    for sz, k in [(tsize, n), (tsize, m), (tsize, m), (4, n), (4, m), (4, m), (4, m), (4, n), (4, n), (4, n),
                  (4, max(n, 128)), (4, 64 * 32), (1, m), (1, n), (1, m), (4, 64)]:
        take(sz, k)
    if csr:
        w2cap = w2 + 64 if w2 else 0
        for sz, k in [(4, s_cap), (4, s_cap), (tsize, s_cap), (4, w2cap), (4, w2cap), (tsize, w2cap)]:
            take(sz, k)
    return off + 16


# ---------------------------------------------------------------------------------------------------------------- cases
# Each case: fn(be, dtype, full) -> Report.  `full` selects the H100 sizes.
FORMS = {"edges": False, "rows": True}      # kernelisation form -> rowwise flag


def _regression_problems():
    """Counterexamples to the old rule (a float key up to half an ulp below its weight, an absolute 2e-6 margin, the comparison
    in the solver's own dtype): name -> (cost, t, optimal x, dtypes whose solver must return exactly that x).  In every one the
    rule must not fire: both rows stay for the augmenting search.
      two_by_two, shared_key -- float64 weights ~1000 whose differences are below half a float key's ulp.  Rounded to float32
        their costs tie, so the float32 solver is held to the optimal objective only.
      f32_sum -- costs and threshold exact in float32, so one problem for both dtypes.  W00 = t - c00 is below
        W01 + W10 by 4.8e-7, less than half a float ulp at 1686: a float32 evaluation of t - c or of the sum of the second-best
        bounds rounds the two sides together and fires the rule on (0, 0)."""
    a = (0.9 - np.array([[1001.00001, 1.0], [1000.00003, -0.05]]), 0.9, [1, 0], (L.F64,))
    b = (0.5 - np.array([[1000.00002], [1000.00003]]), 0.5, [-1, 0], (L.F64,))
    c = (np.array([[-1685.5841064453125, 0.3915400505065918], [-1685.3388671875, np.inf]]), 0.63677978515625, [1, 0], (L.F64, L.F32))
    return {"two_by_two": a, "shared_key": b, "f32_sum": c}


def case_regression(be, dtype, full):
    rep = Report()
    for name, (cost, t, xopt, pinned) in _regression_problems().items():
        for form, rw in FORMS.items():
            x, y, cnt = run_one(be, dtype, cost, t, rowwise=rw)
            obj, opt = check(cost, t, dtype, x, y, rep)
            if dtype in pinned:
                assert list(x) == xopt, "%s/%s: x %s objective %r, optimum %s objective %r" % (name, form, list(x), obj, xopt, opt)
                assert cnt[1] == cost.shape[0], "%s/%s: the rule fixed an edge (rows left %d of %d)" % (name, form, cnt[1], cost.shape[0])
            rep["rounds_" + form] = int(cnt[0])
    return rep


def case_threshold_pairs(be, dtype, full):
    """(0,0) with weight W1 = S_i + S_j + delta against row 0's other edge S_i and column 0's other edge S_j, delta a few float
    ulps (and, in float64, a few double ulps) either side of zero, at weights 2^-10 ... 2^20.  The rule must not fire at
    delta <= 0 (the swap is optimal or tied) and must fire at delta >= 4 float ulps of W1."""
    rep = Report()
    rng = np.random.default_rng(11)
    exps = range(-10, 21) if full else range(-10, 21, 5)
    fired = held = 0
    for e in exps:
        W = 2.0 ** e
        u32 = np.spacing(np.float32(W))
        steps = [-4, -2, -1, 0, 1, 2, 4, 8]
        deltas = [k * float(u32) for k in steps] + ([k * float(np.spacing(W)) for k in (-2, 2)] if dtype == L.F64 else [])
        for d in deltas:
            si = W * float(rng.uniform(0.3, 0.7))
            sj = W - si
            t = 0.5
            cost = np.array([[t - (W + d), t - si], [t - sj, t + 1.0]])
            c, tt = as_dtype(cost, t, dtype)
            true_d = math.fsum([tt, -c[0, 0], -(tt - c[0, 1]), -(tt - c[1, 0])])      # W1 - S_i - S_j of the rounded problem
            for form, rw in FORMS.items():
                x, y, cnt = run_one(be, dtype, cost, t, rowwise=rw)
                check(cost, t, dtype, x, y, rep)
                if true_d <= 0:
                    assert cnt[1] == 2, "rule fired at W1 - S_i - S_j = %r (W ~ 2^%d, %s)" % (true_d, e, form)
                    held += 1
                elif true_d >= 4 * float(np.spacing(np.float32(tt - c[0, 0]))):
                    assert cnt[1] == 0, "rule did not fire at W1 - S_i - S_j = %r (W ~ 2^%d, %s)" % (true_d, e, form)
                    fired += 1
    rep["fired"], rep["held"] = fired, held
    return rep


def case_shared_key(be, dtype, full):
    """Distinct weights that round to one float key: as a column's best (two rows) and as a row's best (two columns).  Either
    edge may be the optimum's, so neither may be fixed."""
    rep = Report()
    for W in ([1.0, 1000.0, 2.0 ** 20] if full else [1000.0]):
        du = float(np.spacing(np.float32(W))) / 8                  # well inside one float key
        t = 0.5
        for cost in (np.array([[t - W], [t - (W + du)]]), np.array([[t - W, t - (W + du)]]),
                     np.array([[t - (W + du), t - W], [t - W, t + 1]])):
            if dtype == L.F32:
                cost = cost.astype(np.float32).astype(np.float64)
            for form, rw in FORMS.items():
                x, y, cnt = run_one(be, dtype, cost, t, rowwise=rw)
                check(cost, t, dtype, x, y, rep)
                if dtype == L.F64:
                    assert cnt[1] == cost.shape[0], "an edge sharing its key with a rival was fixed (%s)" % form
    return rep


def case_negative_costs(be, dtype, full):
    rep = Report()
    rng = np.random.default_rng(3)
    csrs, probs = [], []
    for k in range(60 if full else 16):
        n, m = int(rng.integers(1, 9)), int(rng.integers(1, 9))
        cost = rng.uniform(-200, 0.9, (n, m))
        cost[rng.uniform(size=(n, m)) < 0.4] = 5.0
        c, t = as_dtype(cost, 0.9, dtype)
        csrs.append(R.Csr(n, m, t, R.rows_of(c, t), rowwise=bool(k & 1), poison=False))
        probs.append((cost, 0.9))
    for (cost, t), (x, y, cnt) in zip(probs, solve_csr(be, dtype, csrs)):
        check(cost, t, dtype, x, y, rep)
    return rep


def _chain(K, rng):
    """Path r0-c0-r1-c1-...: (r_i, c_i) weight ~2, (r_{i+1}, c_i) weight ~1.5.  Only the two ends are dominant, so kernelisation
    fixes one pair at each end per round."""
    t = 0.5
    cost = np.full((K, K), t + 1.0)
    for i in range(K):
        cost[i, i] = t - (2.0 + rng.uniform(0, 0.01))
        if i + 1 < K:
            cost[i + 1, i] = t - (1.5 + rng.uniform(0, 0.01))
    return cost, t


def case_chain_round_cap(be, dtype, full):
    rep = Report()
    cost, t = _chain(60 if full else 40, np.random.default_rng(4))
    for form, rw in FORMS.items():
        x, y, cnt = run_one(be, dtype, cost, t, rowwise=rw)
        check(cost, t, dtype, x, y, rep)
        assert cnt[0] == 12 and cnt[1] > 0, "expected the 12-round cap with rows left, got counters %s (%s)" % (list(cnt), form)
        rep["residual_" + form] = int(cnt[1])
    return rep


def _components(c, rng, size=2):
    """c disjoint components of `size` rows x `size` columns that kernelisation cannot touch (every weight ~1, so best < sum of
    second bests); component k owns rows / columns k, k + c, ... so its label is k and it runs on warp k mod 16."""
    n = c * size
    t = 0.5
    cost = np.full((n, n), t + 1.0)
    for k in range(c):
        idx = [k + q * c for q in range(size)]
        for a in idx:
            for b in idx:
                cost[a, b] = t - (1.0 + rng.uniform(0, 0.2))
    return cost, t


def case_component_counts(be, dtype, full):
    rep = Report()
    rng = np.random.default_rng(5)
    for c in (15, 16, 17, 33):
        cost, t = _components(c, rng)
        for form, rw in FORMS.items():
            x, y, cnt = run_one(be, dtype, cost, t, rowwise=rw)
            check(cost, t, dtype, x, y, rep)
            assert cnt[0] == 1 and cnt[1] == 2 * c, "counters %s for %d components (%s)" % (list(cnt), c, form)
    rep["components"] = "15,16,17,33"
    return rep


def case_long_path(be, dtype, full):
    """One component, a path of n rows over n + 1 columns with weights ~1 (weak 0.5 ends): nothing is dominant, and the
    labels have to propagate from row 0 across the whole path."""
    rep = Report()
    n = 1000 if full else 120
    rng = np.random.default_rng(6)
    t = 0.5
    cost = np.full((n, n + 1), t + 1.0)
    for i in range(n):
        cost[i, i] = t - (1.0 + rng.uniform(0, 0.01))
        cost[i, i + 1] = t - (1.0 + rng.uniform(0, 0.01))
    cost[0, 0] = t - 0.5
    cost[n - 1, n] = t - 0.5
    for form, rw in FORMS.items():
        x, y, cnt = run_one(be, dtype, cost, t, rowwise=rw)
        check(cost, t, dtype, x, y, rep, certify=False)
        assert cnt[1] == n, "counters %s (%s)" % (list(cnt), form)
        rep["retries_" + form] = int(cnt[2])
    return rep


def case_frontier_overflow(be, dtype, full):
    """k components of 3 rows over 70 columns each (all pairs eligible, no dominant edge) on warps 0 .. k-1: every search
    outgrows the 64-column frontier, so the single-warp retry queue holds rows of every component at once."""
    rep = Report()
    k = 6 if full else 3
    rng = np.random.default_rng(7)
    R_, Cc = 3, 70
    n, m = k * R_, k * Cc
    t = 0.5
    cost = np.full((n, m), t + 1.0)
    for c in range(k):
        for q in range(R_):
            cost[c + q * k, c * Cc:(c + 1) * Cc] = t - rng.uniform(0.5, 1.0, Cc)
    for form, rw in FORMS.items():
        x, y, cnt = run_one(be, dtype, cost, t, rowwise=rw)
        check(cost, t, dtype, x, y, rep)
        assert cnt[1] == n and cnt[2] >= k, "counters %s (%s)" % (list(cnt), form)
        rep["retries_" + form] = int(cnt[2])
    return rep


def case_single_retry(be, dtype, full):
    """Exactly one search outgrows its frontier: row 0 over 70 columns, row 1 sharing row 0's best column."""
    rep = Report()
    rng = np.random.default_rng(8)
    t = 0.5
    cost = np.full((2, 70), t + 1.0)
    cost[0] = t - rng.uniform(0.5, 0.6, 70)
    cost[0, 0] = t - 1.0
    cost[1, 0] = t - 0.9
    for form, rw in FORMS.items():
        x, y, cnt = run_one(be, dtype, cost, t, rowwise=rw)
        check(cost, t, dtype, x, y, rep)
        assert cnt[2] == 1, "counters %s (%s)" % (list(cnt), form)
    return rep


def case_dense(be, dtype, full):
    """Every pair eligible (t above every cost), through both entries."""
    rep = Report()
    rng = np.random.default_rng(9)
    shapes = [(512, 512), (1, 4096), (4096, 1)] if full else [(48, 48), (1, 512), (512, 1)]
    for n, m in shapes:
        cost = rng.uniform(0, 1, (n, m))
        t = 1.5
        x, y = solve_dense(be, dtype, cost, t)
        check(cost, t, dtype, x, y, rep, certify=n <= 64)
        x2, y2, cnt = run_one(be, dtype, cost, t)
        assert np.array_equal(x, x2) and np.array_equal(y, y2), "the CSR entry disagrees with the dense entry at %dx%d" % (n, m)
    return rep


def _storage_problem(full, seed):
    rng = np.random.default_rng(seed)
    n, m = (90, 70) if full else (40, 30)
    t = 0.9
    cost = rng.uniform(0, 1.4, (n, m))
    cost[rng.uniform(size=(n, m)) < 0.8] = 5.0
    cost[rng.integers(0, n, 3)] = 5.0                          # empty rows
    rows = R.rows_of(cost, t, rng, pad=0.3, shuffle=True)
    return cost, t, rows


def case_storage(be, dtype, full, only=None):
    """Every placement of the shared-memory mirror and the second window, in both kernelisation forms, one batch: each result
    must equal the same problem with everything in global memory, bit for bit, and be optimal."""
    rep = Report()
    cost, t, rows = _storage_problem(full, 10)
    c, tt = as_dtype(cost, t, dtype)
    rows = [[(j, float(npdt(dtype)(v))) for j, v in r] for r in rows]
    n, m = cost.shape
    pl = R.placements(rows)
    csrs, names = [], []
    for name, (s_cap, w2) in pl.items():
        if only and name not in only:
            continue
        for form, rw in FORMS.items():
            csrs.append(R.Csr(n, m, tt, rows, s_cap, w2, rw, seed=len(csrs)))
            names.append((name, form))
            csrs.append(R.Csr(n, m, tt, rows, 0, (0, 0), rw, poison=False))
            names.append(("plain", form))
    res = solve_csr(be, dtype, csrs)
    ref = R.certify(c, tt)
    for k in range(0, len(csrs), 2):
        (x, y, cnt), (x0, y0, cnt0) = res[k], res[k + 1]
        check(cost, t, dtype, x0, y0, rep, ref=ref)
        check(cost, t, dtype, x, y, rep, ref=ref)
        assert np.array_equal(x, x0) and np.array_equal(y, y0) and np.array_equal(cnt, cnt0), \
            "placement %s/%s differs from global storage: counters %s vs %s" % (names[k] + (list(cnt), list(cnt0)))
    rep["placements"] = len(csrs) // 2
    return rep


def case_degenerate(be, dtype, full):
    rep = Report()
    t = 0.7
    probs = [np.zeros((0, 5)), np.zeros((5, 0)), np.zeros((0, 0)), np.array([[0.1]]), np.array([[0.7]]),
             np.full((1, 6), 0.3), np.full((6, 1), 0.3), np.full((4, 4), 0.9),             # everything gated
             np.full((3, 3), t),                                                           # cost == t is excluded
             np.array([[np.inf, 0.2, np.nan], [np.nan, np.inf, 0.1], [0.3, np.nan, -5.0]]),
             np.array([[-0.0, 0.5], [0.5, -0.0]]),
             np.full((4, 5), 0.25),                                                        # ties: any valid matching
             np.array([[0.1, 0.1, 0.6], [0.1, 0.1, 0.6]])]
    for cost in probs:
        n, m = cost.shape
        x, y = solve_dense(be, dtype, cost, t)
        check(cost, t, dtype, x, y, rep)
        if n * m:
            x2, y2, cnt = run_one(be, dtype, cost, t)
            check(cost, t, dtype, x2, y2, rep)
        if np.all(~R.eligible(cost, t)):
            assert np.all(x == -1) and np.all(y == -1)
    return rep


def case_tiny_weights(be, dtype, full):
    """Float64 weights below half of float32's smallest denormal: their float keys round to 0, which must not read as "no edge"
    (the edge-parallel form would drop the row).  The rule cannot separate such weights, so every row goes to the search."""
    rep = Report()
    if dtype != L.F64:
        return rep                  # (a float32 weight t - c > 0 is at least the smallest denormal)
    t = 1e-300
    for cost in (np.array([[0.0]]), np.array([[0.0, 5e-301], [4e-301, 8e-301]]), np.array([[0.0, 5e-301, -2e-300]])):
        for form, rw in FORMS.items():
            x, y, cnt = run_one(be, dtype, cost, t, rowwise=rw)
            check(cost, t, dtype, x, y, rep)
            assert cnt[1] == cost.shape[0], "%s: counters %s" % (form, list(cnt))
    return rep


def case_row_index_optional(be, dtype, full):
    """Row-parallel problems read no row index: e_row = m_row = NULL with the shared mirror and the second window in use solves
    them as with the indices given.  An edge-parallel problem without row indices is B2T_EINVAL, nothing launched."""
    rep = Report()
    cost, t, rows = _storage_problem(full, 14)
    rows = [[(j, float(npdt(dtype)(v))) for j, v in r] for r in rows]
    n, m = cost.shape
    placed = [R.Csr(n, m, t, rows, s_cap, w2, True, poison=False) for s_cap, w2 in R.placements(rows).values()]
    with_idx = solve_csr(be, dtype, placed, mirrors=False)
    without = solve_csr(be, dtype, placed, mirrors=False, row_index=False)
    for a, b in zip(with_idx, without):
        for u, v in zip(a, b):
            assert np.array_equal(u, v), "a row-parallel solve changed without row indices"
        check(cost, t, dtype, b[0], b[1], rep)
    solve_csr(be, dtype, [R.Csr(n, m, t, rows, 0, (0, 0), False, poison=False)], expect_rc=L.EINVAL, mirrors=False, row_index=False)
    rep["placements"] = len(placed)
    return rep


def largest_square(tsize, csr, limit=227 * 1024):
    n = 1
    while lap_smem_bytes(n + 1, n + 1, tsize, csr) <= limit:
        n += 1
    return n


def _band(N, t, rng):
    cost = np.full((N, N), t + 1.0)
    d = np.arange(N)
    cost[d, d] = t - rng.uniform(0.5, 1.0, N)
    cost[d[1:], d[:-1]] = t - rng.uniform(0.5, 1.0, N - 1)        # a tie-free bidiagonal band
    return cost


def case_limits(be, dtype, full):
    """The largest n = m that fits 227 KB of shared memory solves, through each entry; one more is B2T_ECAPACITY, unlaunched."""
    rep = Report()
    ts = 8 if dtype == L.F64 else 4
    rng = np.random.default_rng(12)
    t = 0.5
    N = largest_square(ts, True)
    cost = _band(N, t, rng)
    x2, y2, cnt = run_one(be, dtype, cost, t)
    check(cost, t, dtype, x2, y2, rep, certify=False)
    solve_csr(be, dtype, [R.Csr(N + 1, N + 1, t, [[] for _ in range(N + 1)])], expect_rc=L.ECAPACITY)
    Nd = largest_square(ts, False)
    if full:                        # (the simulator would spend minutes in the dense entry's N x N sparsify pass)
        cost = _band(Nd, t, rng)
        x, y = solve_dense(be, dtype, cost, t)
        check(cost, t, dtype, x, y, rep, certify=False)
    solve_dense(be, dtype, np.full((Nd + 1, Nd + 1), t + 1.0), t, expect_rc=L.ECAPACITY)
    rep["N_csr"], rep["N_dense"] = N, Nd
    return rep


def case_batch(be, dtype, full):
    """64 differently shaped problems in one launch (placements and forms mixed), each bitwise equal to its single solve, and
    the whole launch repeated once: identical."""
    rep = Report()
    rng = np.random.default_rng(13)
    csrs, costs = [], []
    for k in range(64 if full else 12):
        n, m = int(rng.integers(0, 40)), int(rng.integers(0, 40))
        t = 0.9
        cost = rng.uniform(-1, 1.2, (n, m))
        c, tt = as_dtype(cost, t, dtype)
        rows = R.rows_of(c, tt, rng, pad=0.2)
        pl = list(R.placements(rows).values())
        s_cap, w2 = pl[k % len(pl)]
        csrs.append(R.Csr(n, m, tt, rows, s_cap, w2, bool(k & 1), seed=k))
        costs.append((cost, t))
    res = solve_csr(be, dtype, csrs)
    again = solve_csr(be, dtype, csrs)
    for k, c in enumerate(csrs):
        single = solve_csr(be, dtype, [c])[0]
        for a, b in zip(res[k], single):
            assert np.array_equal(a, b), "problem %d of the batch differs from its single solve" % k
        for a, b in zip(res[k], again[k]):
            assert np.array_equal(a, b), "problem %d differs between two identical launches" % k
        check(costs[k][0], costs[k][1], dtype, res[k][0], res[k][1], rep)
    return rep


CASES = {
    "regression": case_regression,
    "threshold_pairs": case_threshold_pairs,
    "shared_key": case_shared_key,
    "negative_costs": case_negative_costs,
    "chain_round_cap": case_chain_round_cap,
    "component_counts": case_component_counts,
    "long_path": case_long_path,
    "frontier_overflow": case_frontier_overflow,
    "single_retry": case_single_retry,
    "dense": case_dense,
    "storage": case_storage,
    "degenerate": case_degenerate,
    "limits": case_limits,
    "tiny_weights": case_tiny_weights,
    "row_index_optional": case_row_index_optional,
    "batch": case_batch,
}
