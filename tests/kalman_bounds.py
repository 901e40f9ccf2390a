"""TEST INFRASTRUCTURE: seeded edge inputs and per-entry-point checks of the standalone Kalman / IoU entry points against
tests/kalman_ref.py, shared by tests/test_gpu_kalman_bounds.py (nvcc build, through b200track.engine.Ops) and
tests/test_hostsim_kalman_bounds.py (the same source under the host simulator).  A backend is an object with the methods
initiate / predict / project / update / gating / gmc / iou taking and returning NumPy arrays in the kernel's dtype.

Inputs: centres up to 8192, heights 1 - 4000 px (1 - 2 px included), aspect ratios 0.02 - 50, covariances after 1, 30 and 300
predict-only steps from initiate (and one update, so that every entry of the 8 x 8 matrix is populated), NSA confidences in
{0, 0.5, 0.99, 0.999, nextafter(1, 0)}, warps with rotation up to 5 degrees and scale 0.9 - 1.1."""
import numpy as np

import kalman_ref as R
from b200track._lib import FLAG_MEAN_F32, FLAG_NOT_TRACKED
from oracle import kalman as K

FMTS = {"xyah": K.FMT_XYAH, "xywh": K.FMT_XYWH, "nsa": K.FMT_NSA}
COUNTS = [1, 3, 4, 5, 127, 128, 129, 4097]
CONFS = np.array([0.0, 0.5, 0.99, 0.999, np.nextafter(np.float32(1), np.float32(0))], np.float32)
STEPS = (1, 30, 300)


def measurements(rng, n, fmt, mild=False):
    """(n, 4) float32 measurements (x, y, a, h) or (x, y, w, h) at the edges (mild: 20 - 300 px, aspect 0.3 - 3)."""
    xy = rng.uniform(0, 8192, (n, 2))
    if mild:
        h = rng.uniform(20, 300, n)
        ar = rng.uniform(0.3, 3.0, n)
    else:
        h = np.exp(rng.uniform(np.log(1.0), np.log(4000.0), n))
        h[: max(1, n // 8)] = rng.uniform(1.0, 2.0, max(1, n // 8))               # 1 - 2 px boxes
        ar = np.exp(rng.uniform(np.log(0.02), np.log(50.0), n))
    w = ar * h
    third = w if fmt == K.FMT_XYWH else ar
    return np.stack([xy[:, 0], xy[:, 1], third, h], 1).astype(np.float32)


def states(rng, n, fmt, mild=False):
    """(mean (n, 8), cov (n, 8, 8)) float64 via the oracle: initiate, one update, then 1 / 30 / 300 predicts (mild: 30)."""
    z = measurements(rng, n, fmt, mild)
    m, c = zip(*[K.initiate(fmt, zi) for zi in z])
    mean = np.stack(m).astype(np.float64)
    cov = np.stack(c).astype(np.float64)
    mean, cov = K.multi_predict(fmt, mean, cov)
    zk = z + (rng.normal(0, 1, z.shape) * np.array([1, 1, 0.01, 0.5]) * (z[:, 3:4] / 50 + 0.1)).astype(np.float32)
    zk[:, 2:] = np.abs(zk[:, 2:]) + np.float32(0.01)
    for i in range(n):
        mean[i], cov[i] = K.update(fmt, mean[i], cov[i], zk[i].astype(np.float64))
    steps = np.full(n, 30) if mild else rng.choice(STEPS, n)
    for k in range(int(steps.max())):
        sel = steps > k
        mean[sel], cov[sel] = K.multi_predict(fmt, mean[sel], cov[sel])
    cov = 0.5 * (cov + cov.transpose(0, 2, 1))
    return mean, cov


def near(rng, mean, fmt, scale=1.0):
    """(n, 4) float32 measurements near each state's projected mean."""
    n = len(mean)
    h = np.abs(mean[:, 3:4])
    noise = rng.normal(0, 1, (n, 4)) * np.array([0.1, 0.1, 0.01, 0.05]) * (h if fmt == K.FMT_XYWH else np.concatenate(
        [h, h, np.ones((n, 1)), h], 1)) * scale
    z = (mean[:, :4] + noise).astype(np.float32)
    z[:, 2:] = np.maximum(np.abs(z[:, 2:]), np.float32(0.01))
    return z


def warps(rng, k):
    """k (2, 3) similarity warps: rotation up to +-5 degrees, scale 0.9 - 1.1, shifts up to 40 px."""
    out = []
    for _ in range(k):
        a = np.deg2rad(rng.uniform(-5, 5))
        s = rng.uniform(0.9, 1.1)
        out.append(np.array([[s * np.cos(a), -s * np.sin(a), rng.uniform(-40, 40)],
                             [s * np.sin(a), s * np.cos(a), rng.uniform(-40, 40)]]))
    return out


def _dt(f32):
    return np.float32 if f32 else np.float64


def _check_state(nm, nP, got_m, got_c, f32, what, stats):
    r = max(R.check(got_m, R.stack(nm), f32, what + " mean"), R.check(got_c, R.stack_cov(nP), f32, what + " cov"))
    stats[what.split(" ")[0]] = max(stats.get(what.split(" ")[0], 0.0), r)
    return r


def _vs_oracle(om, oc, gm, gc, rm, rc, what):
    """float64: oracle/kalman.py (NumPy / LAPACK, pinned bit for bit to the reference) evaluates the same operations in another order,
    so it and the kernel both lie within the bound of the exact value: |kernel - oracle| <= 2 x bound.  This also pins the
    restatement's float32-quirk branches to the oracle's."""
    for o, g, r, part in ((om, gm, rm, "mean"), (oc, gc, rc, "cov")):
        if o is None:
            continue
        d = np.abs(np.asarray(o, np.float64) - np.asarray(g, np.float64))
        b = 2 * R.bound_any_order(r, False)
        assert (d <= b).all(), "%s %s: the float64 kernel and the oracle differ by more than twice the bound (%.3g)" % (
            what, part, float((d / b).max()))


# ---------------------------------------------------------------- per-entry-point checks
def run_entry_points(be, fmt, f32, n, seed, stats, mild=False):
    """Every standalone entry point at n tracks; stats[name] collects the largest err / bound.  mild: also assert the bound
    cap (kalman_ref.cap_ok).  Returns nothing; raises AssertionError on the first failure."""
    rng = np.random.default_rng(seed)
    dt = _dt(f32)
    tag = "%s %s n=%d" % ("f32" if f32 else "f64", [k for k, v in FMTS.items() if v == fmt][0], n)
    mean, cov = states(rng, n, fmt, mild)
    mean, cov = mean.astype(dt), cov.astype(dt)

    # initiate
    z0 = measurements(rng, n, fmt, mild)
    gm, gc = be.initiate(fmt, z0.astype(dt))
    im, iP = R.kf_initiate(z0, fmt, f32)
    _check_state(im, iP, gm, gc, f32, "initiate " + tag, stats)
    if mild:
        R.cap_ok(R.stack_cov(iP), f32, "initiate " + tag)
    if not f32:
        for i in range(n):
            om, oc = K.initiate(fmt, z0[i])
            _vs_oracle(om, oc, gm[i], gc[i], R.stack(im).take(i), R.stack_cov(iP).take(i), "initiate %s track %d" % (tag, i))

    # predict: flags NOT_TRACKED on every other track, q_f32 both ways (the initiate output is the q_f32 case's state)
    zero_vh = (np.arange(n) % 2) == 1
    flags = np.where(zero_vh, FLAG_NOT_TRACKED, 0).astype(np.int32)
    for q_f32, (m0, c0) in ((False, (mean, cov)), (True, (gm.astype(dt), gc.astype(dt)))):
        pm, pc = be.predict(fmt, m0, c0, flags, q_f32)
        m, P = R.state(m0, c0, f32)
        nm, nP = R.kf_predict(m, P, fmt, zero_vh, q_f32, f32)
        _check_state(nm, nP, pm, pc, f32, "predict %s q_f32=%d" % (tag, q_f32), stats)
        if mild:
            R.cap_ok(R.stack_cov(nP), f32, "predict " + tag)
        if not f32:
            mz = m0.copy()
            mz[zero_vh, 7] = 0
            om, oc = K.multi_predict(fmt, mz.astype(np.float32) if q_f32 else mz, c0, all_f32=q_f32)
            _vs_oracle(om, oc, pm, pc, R.stack(nm), R.stack_cov(nP), "predict %s q_f32=%d" % (tag, q_f32))

    # project and update: mean_f32 on every third track, NSA confidences cycling through CONFS
    mf = (np.arange(n) % 3) == 2
    pflags = np.where(mf, FLAG_MEAN_F32, 0).astype(np.int32)
    conf = CONFS[np.arange(n) % len(CONFS)] if fmt == K.FMT_NSA else None
    if mild and conf is not None:
        conf = np.full(n, 0.5, np.float32)
    m, P = R.state(mean, cov, f32)
    zm, zc = be.project(fmt, mean, cov, pflags, conf)
    S = R.innovation_cov(m, P, fmt, mf, conf, f32)
    r = max(R.check(zm, R.stack(m[:4]), f32, "project %s mean" % tag), R.check(zc, R.stack_cov(S), f32, "project %s cov" % tag))
    stats["project"] = max(stats.get("project", 0.0), r)
    if mild:
        R.cap_ok(R.stack_cov(S), f32, "project " + tag)
    if not f32:
        for i in range(n):
            zh, so = K.project(fmt, mean[i], cov[i], bool(mf[i]), 0.0 if conf is None else conf[i])
            _vs_oracle(zh, so, zm[i], zc[i], R.stack(m[:4]).take(i), R.stack_cov(S).take(i), "project %s track %d" % (tag, i))

    # update through idx: every other row, last first; the rows it does not name must not change
    idx = np.arange(n)[::-1][::2].copy().astype(np.int32)
    k = len(idx)
    zu = near(rng, mean[idx], fmt).astype(dt)
    ck = None if conf is None else conf[:k].copy()
    um, uc = be.update(fmt, mean, cov, idx, zu, ck, pflags[:k].copy())
    rest = np.setdiff1d(np.arange(n), idx)
    assert np.array_equal(um[rest], mean[rest]) and np.array_equal(uc[rest], cov[rest]), "update %s: a row outside idx changed" % tag
    ms, Ps = R.state(mean[idx], cov[idx], f32)
    zb = [R.inputs(zu[:, q], f32) for q in range(4)]
    nm, nP = R.kf_update(ms, Ps, fmt, zb, mf[:k], ck, f32)
    _check_state(nm, nP, um[idx], uc[idx], f32, "update " + tag, stats)
    if mild:
        R.cap_ok(R.stack(nm), f32, "update %s mean" % tag)
        R.cap_ok(R.stack_cov(nP), f32, "update %s cov" % tag)

    # gmc
    w = warps(rng, 1)[0]
    wk = w.reshape(-1).astype(dt)
    gmm, gmc = be.gmc(mean, cov, w)
    m, P = R.state(mean, cov, f32)
    nm, nP = R.kf_gmc(m, P, wk)
    _check_state(nm, nP, gmm, gmc, f32, "gmc " + tag, stats)
    if mild:
        R.cap_ok(R.stack_cov(nP), f32, "gmc " + tag)
    if not f32:
        om, oc = K.gmc_apply(mean, cov, w)
        _vs_oracle(om, oc, gmm, gmc, R.stack(nm), R.stack_cov(nP), "gmc " + tag)

    # gating: a few states against every measurement, both metrics and both only_position values
    zg = np.concatenate([near(rng, mean, fmt, 3.0), measurements(rng, n, fmt, mild)]).astype(dt)
    for i in sorted({0, n // 2, n - 1}):
        for mean_f32 in (False, True):
            for op in (False, True):
                for metric in (0, 1):
                    got = be.gating(fmt, mean[i], cov[i], zg, op, metric, mean_f32)
                    ref = R.gating(fmt, mean[i], cov[i], zg, op, metric, f32, mean_f32)
                    r = R.check(got, ref, f32, "gating %s state %d mean_f32=%d only_position=%d metric=%d" % (tag, i, mean_f32, op, metric))
                    stats["gating"] = max(stats.get("gating", 0.0), r)
                    if mild:
                        R.cap_ok(ref, f32, "gating %s state %d" % (tag, i))
                    if not f32:
                        o = K.gating_distance(fmt, mean[i], cov[i], zg, op, "maha" if metric == 0 else "gaussian", mean_f32)
                        _vs_oracle(o, None, got, None, ref, None, "gating %s state %d" % (tag, i))


def iou_boxes(rng, n, scale, smax):
    """(n, 4) tlbr: corners up to `scale`, sizes 1 - smax px, half of them on half-pixel grids."""
    p = rng.uniform(0, scale, (n, 2))
    s = np.exp(rng.uniform(0, np.log(smax), (n, 2)))
    if smax > 4096:                                                      # some single +1 areas past 2^24
        s[: max(1, n // 8)] = rng.uniform(4200, smax, (max(1, n // 8), 2))
    b = np.concatenate([p, p + s], 1)
    b[::2] = np.round(b[::2] * 2) / 2
    return b.astype(np.float32)


def run_iou(be, f32, n, m, seed, stats):
    """iou_cost against kalman_ref.iou_plus1, as IoU and as distance: at 1280 px frames with boxes of 1 - 4000 px, and at 8K
    coordinates with boxes up to 8000 px, whose single +1 areas pass 2^24 (asserted).  On the 1280 px frames the bound is also held
    below the cap."""
    rng = np.random.default_rng(seed)
    dt = _dt(f32)
    for scale, smax in ((1280.0, 4000.0), (8192.0, 8000.0)):
        a = iou_boxes(rng, n, scale, smax)
        b = np.concatenate([a[rng.integers(0, n, m // 2)] + rng.normal(0, 2, (m // 2, 4)).astype(np.float32),
                            iou_boxes(rng, m - m // 2, scale, smax)]).astype(np.float32)
        b[:, 2:] = np.maximum(b[:, 2:], b[:, :2])
        a, b = a.astype(dt), b.astype(dt)
        ref, amb = R.iou_plus1(a, b, f32)
        if scale > 4096 and n * m >= 64:
            areas = np.concatenate([(a[:, 2] - a[:, 0] + 1.0) * (a[:, 3] - a[:, 1] + 1.0), (b[:, 2] - b[:, 0] + 1.0) * (b[:, 3] - b[:, 1] + 1.0)])
            assert areas.max() > 2.0 ** 24, "no single +1 area passes 2^24"
        if scale < 4096:
            nz = (ref.v > 0) & ~amb
            R.cap_ok(R.B(ref.v[nz], ref.u, ref.e[nz], ref.m[nz]), f32, "iou_cost n=%d m=%d" % (n, m))
        for as_distance in (0, 1):
            got = be.iou(a, b, as_distance)
            if as_distance:
                ref_d = R.const(1.0, f32, ref.u) - ref
                ok = ~amb
                r = R.check(got[ok], R.B(ref_d.v[ok], ref.u, ref_d.e[ok]), f32, "iou_cost f%d n=%d m=%d scale %g distance" % (
                    32 if f32 else 64, n, m, scale))
                assert np.all((got[amb] == 1) | (np.abs(got[amb] - ref_d.v[amb].astype(np.float64)) <= R.bound(ref_d, f32)[amb]))
            else:
                ok = ~amb
                r = R.check(got[ok], R.B(ref.v[ok], ref.u, ref.e[ok]), f32, "iou_cost f%d n=%d m=%d scale %g" % (
                    32 if f32 else 64, n, m, scale))
                assert np.all((got[amb] == 0) | (np.abs(got[amb] - ref.v[amb].astype(np.float64)) <= R.bound(ref, f32)[amb]))
            stats["iou_cost"] = max(stats.get("iou_cost", 0.0), r)

