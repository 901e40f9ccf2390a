"""TEST INFRASTRUCTURE: one iteration of the ECC kernel (csrc/b2t_ecc.cu ``ecc_iterate_kernel`` + ``ecc_step``) with a derived bound,
shared by the GPU tier (tests/test_gpu_ecc_stages.py) and the CPU tier (tests/test_hostsim_ecc_stages.py).

Given the template, the current plane and the map the iteration starts from (the device's own map of the previous iteration),
``step_set`` returns every map (float32 bit patterns) and flag the kernel can reach, and an interval that holds its rho.

Sums.  Every one of the 21 terms is exact in fp64: a product of two fp32 values, or of an fp32 value and a uint8 (the warped
planes come from ``oracle/ecc.py``, which is bit-exact with cv2.warpAffine and with the kernel's warp stage).  So the kernel and any
reference differ only in summation order.  Each sum is taken correctly rounded (``math.fsum``); the kernel's sum lies within
    gamma_D * sum|t| + ulp(fsum) / 2,     gamma_D = D u / (1 - D u),  u = 2^-53,
where D is the kernel's own reduction depth: ceil(pixels per CTA / 512) sequential adds per thread, 5 butterfly levels, 16 warps in
order and C CTAs in rank order (C = 8 on the GPU, 1 in the simulator).  A sum whose terms all lie on a grid 2^-g with
sum|t| < 2^(53 - g) (the mask count, the template sums, the warped image sums at moderate sizes) is exact in any order: bound 0.

Step.  ``ecc_step`` is restated in its own operation order on ``V`` values: the reference value ``v`` (an IEEE double computed by
the same operation on the reference's operands) and a first-order bound ``r`` on |kernel - v|:
  a +- b : ra + rb                    a * b : |a| rb + |b| ra + ra rb          a / b : (ra + |a / b| rb) / (|b| - rb)
  sqrt a : min(ra / sqrt(a), sqrt(ra))
each plus u (2 |v| + r) for the two roundings; an operation whose operands are exact (r = 0) is the kernel's own operation: r = 0.
cos / sin / asin carry the device's documented maximum error for double (CUDA Math API: 2 ulp each) plus 1 ulp for the host's
libm; in the simulator the kernel calls the same libm (1 ulp).  At each rounding to float32 (the masked means, the Hessian, its
inverse, the projections, Hi ip, ep, dp, the map update, cos, sin) either no float32 rounding boundary lies inside [v - r, v + r] --
the rounded value is determined, r = 0 -- or the value forks into both float32 neighbours.  The decisions lambda_d <= 0, NaN rho and
|rho - last| < eps fork the same way when undecided.  More than ``MAX_FORKS`` forks in one iteration, or an interval wider than two
float32 values, raises ``BoundTooLoose``: a bound that loose would not test anything."""
import math

import numpy as np

from oracle import ecc as E

U = 2.0 ** -53
MAX_FORKS = 8
ULP_DEVICE = 2            # CUDA Math API, double precision: max ulp error of sin, cos, asin
ULP_HOST = 1
KTHREADS, KWARPS = 512, 16
CONTINUE = 0              # a completed update that did not converge (the caller's ITER_CAP when it was the last allowed)


class BoundTooLoose(AssertionError):
    pass


def depth(h, w, cluster):
    """The kernel's reduction depth: the most additions any one term goes through on its way into a sum."""
    total = h * w
    per_cta = max((total * (r + 1)) // cluster - (total * r) // cluster for r in range(cluster))
    return -(-per_cta // KTHREADS) + 5 + KWARPS + cluster


def terms(tmpl, img, M):
    """The 21 term arrays in the kernel's order: n, SI, SII, ST, STT, STI over the mask; SJI (3) over all pixels; SJ, SJT (3 each)
    over the mask; SJJ 00 01 02 11 12 22 over all pixels.  fp64 arrays whose every element is exact."""
    h, w = tmpl.shape
    gx, gy = E.gradients(img)
    I = E.warp_linear(img.astype(np.float32), M)
    GX, GY = E.warp_linear(gx, M), E.warp_linear(gy, M)
    m = E.warp_nearest_mask(h, w, M).astype(bool)
    c, s = np.float32(M[0][0]), np.float32(M[1][0])
    ys, xs = np.mgrid[0:h, 0:w].astype(np.float32)
    J = [(GX * (-(xs * s) - (ys * c)) + GY * (xs * c - ys * s)).astype(np.float64), GX.astype(np.float64), GY.astype(np.float64)]
    I, T = I.astype(np.float64), tmpl.astype(np.float64)
    out = [np.ones(int(m.sum())), I[m], (I * I)[m], T[m], (T * T)[m], (T * I)[m]]
    out += [j * I for j in J] + [j[m] for j in J] + [(j * T)[m] for j in J]
    out += [J[a] * J[b] for a, b in ((0, 0), (0, 1), (0, 2), (1, 1), (1, 2), (2, 2))]
    return [np.ascontiguousarray(t).ravel() for t in out]


def _on_grid(t, total_abs):
    """True when every partial sum of t, in any order, is an fp64 value: all terms are multiples of one 2^g and sum|t| < 2^(g+53)."""
    nz = t[t != 0]
    if nz.size == 0:
        return True
    mant, ex = np.frexp(nz)
    mi = np.abs((mant * 2.0 ** 53).astype(np.int64))
    low = mi & -mi
    g = int((ex.astype(np.int64) - 53 + np.round(np.log2(low.astype(np.float64))).astype(np.int64)).min())
    return total_abs < 2.0 ** (g + 53)


def sums_with_bound(tmpl, img, M, cluster):
    """(sums, bounds): each of the 21 sums correctly rounded, and the bound on the kernel's depth-D sum around it."""
    D = depth(*tmpl.shape, cluster)
    gam = D * U / (1 - D * U)
    S, R = [], []
    for t in terms(tmpl, img, M):
        s = math.fsum(t.tolist())
        a = math.fsum(np.abs(t).tolist())
        S.append(s)
        R.append(0.0 if _on_grid(t, a) else (gam * a * (1 + 2 * U) + math.ulp(s) / 2))
    return S, R


# ---------------------------------------------------------------------------------------------- values with a running bound
class V:
    __slots__ = ("v", "r")

    def __init__(self, v, r=0.0):
        self.v, self.r = float(v), float(r)

    @staticmethod
    def _mk(v, rp):
        if rp == 0.0:
            return V(v, 0.0)
        return V(v, (rp + U * (2 * abs(v) + rp)) * (1 + 2.0 ** -40))

    def __add__(self, o):
        o = _v(o)
        return V._mk(self.v + o.v, self.r + o.r)

    def __radd__(self, o):
        return _v(o) + self

    def __sub__(self, o):
        o = _v(o)
        return V._mk(self.v - o.v, self.r + o.r)

    def __rsub__(self, o):
        return _v(o) - self

    def __mul__(self, o):
        o = _v(o)
        return V._mk(self.v * o.v, abs(self.v) * o.r + abs(o.v) * self.r + self.r * o.r)

    def __rmul__(self, o):
        return _v(o) * self

    def __truediv__(self, o):
        o = _v(o)
        if o.r == 0.0 and o.v == 0.0:
            raise ZeroDivisionError
        if abs(o.v) <= o.r:
            raise BoundTooLoose("divisor interval holds 0")
        q = self.v / o.v
        return V._mk(q, 0.0 if self.r == 0.0 and o.r == 0.0 else (self.r + abs(q) * (1 + 2 * U) * o.r) / (abs(o.v) - o.r))

    def lo(self):
        return math.nextafter(self.v - self.r, -math.inf) if self.r else self.v

    def hi(self):
        return math.nextafter(self.v + self.r, math.inf) if self.r else self.v


def _v(x):
    return x if isinstance(x, V) else V(x)


def vsqrt(a):
    if a.v < 0.0:                                                 # the positive branch of a variance interval that straddles 0
        raise BoundTooLoose("sqrt of an interval centred below 0")
    s = math.sqrt(a.v)
    if a.r == 0.0:
        return V(s)
    rp = min(a.r / s if s > 0 else math.inf, math.sqrt(a.r))
    return V._mk(s, rp)


def f32(x):
    return float(np.float32(x))


class _Path:
    """One path through the forks: ``choose`` replays a recorded choice, or takes 0 and records the new fork."""

    def __init__(self, choices):
        self.choices, self.pos, self.widths = list(choices), 0, []

    def choose(self, n):
        if self.pos == len(self.choices):
            self.choices.append(0)
        c = self.choices[self.pos]
        self.widths.append(n)
        self.pos += 1
        return c

    def f32(self, x):
        """(float) x: determined, or one of the two float32 neighbours around the interval."""
        if x.r == 0.0:
            return V(f32(x.v))
        a, b = np.float32(x.lo()), np.float32(x.hi())
        if a == b:
            return V(float(a))
        if np.nextafter(a, np.float32(np.inf)) != b:
            raise BoundTooLoose("interval [%r, %r] spans more than two float32 values" % (x.lo(), x.hi()))
        return V(float((a, b)[self.choose(2)]))

    def test(self, lo_true, hi_true):
        """A decision that holds on the whole interval (lo_true), on none of it (not hi_true), or forks."""
        if lo_true == hi_true:
            return lo_true
        return bool(self.choose(2))

    def fn(self, f, df_max, x, ulps):
        v = f(x.v)
        return V(v, (df_max * x.r + ulps * math.ulp(abs(v) + x.r)) * (1 + 2.0 ** -40))


def _step(p, S, Mf, last, eps, ulps):
    """ecc_step + the convergence test of ecc_iterate_kernel on one path.  S: 21 V sums; Mf: the float32 map (m00 m01 m02 m10 m11
    m12).  Returns (map, flag, rho)."""
    n = S[0]
    im, tm = S[1] / n, S[3] / n
    iv, tv = S[2] / n - im * im, S[4] / n - tm * tm
    istd = vsqrt(iv if p.test(iv.lo() > 0.0, iv.hi() > 0.0) else V(0.0))
    tstd = vsqrt(tv if p.test(tv.lo() > 0.0, tv.hi() > 0.0) else V(0.0))
    imf, tmf = p.f32(im), p.f32(tm)
    tnorm, inorm = vsqrt(n * tstd * tstd), vsqrt(n * istd * istd)
    h = [p.f32(S[k]) for k in range(15, 21)]
    m = [[h[0], h[1], h[2]], [h[1], h[3], h[4]], [h[2], h[4], h[5]]]
    d = m[0][0] * (m[1][1] * m[2][2] - m[1][2] * m[2][1]) - m[0][1] * (m[1][0] * m[2][2] - m[1][2] * m[2][0]) + \
        m[0][2] * (m[1][0] * m[2][1] - m[1][1] * m[2][0])
    assert d.r == 0.0                                             # the Hessian is float32 on every path: d is the kernel's own
    if d.v != 0.0:
        d = V(1.0 / d.v)
        Hi = [[p.f32((m[1][1] * m[2][2] - m[1][2] * m[2][1]) * d), p.f32((m[0][2] * m[2][1] - m[0][1] * m[2][2]) * d),
               p.f32((m[0][1] * m[1][2] - m[0][2] * m[1][1]) * d)],
              [p.f32((m[1][2] * m[2][0] - m[1][0] * m[2][2]) * d), p.f32((m[0][0] * m[2][2] - m[0][2] * m[2][0]) * d),
               p.f32((m[0][2] * m[1][0] - m[0][0] * m[1][2]) * d)],
              [p.f32((m[1][0] * m[2][1] - m[1][1] * m[2][0]) * d), p.f32((m[0][1] * m[2][0] - m[0][0] * m[2][1]) * d),
               p.f32((m[0][0] * m[1][1] - m[0][1] * m[1][0]) * d)]]
    else:
        Hi = [[V(0.0)] * 3 for _ in range(3)]
    corr = S[5] - imf * S[3] - tmf * S[1] + n * tmf * imf
    den = inorm * tnorm
    if den.r == 0.0 and den.v == 0.0:
        rho = V(math.nan) if corr.r == 0.0 and corr.v == 0.0 else None
        if rho is None:
            if corr.lo() <= 0.0 <= corr.hi():
                raise BoundTooLoose("rho = corr / 0 with the sign of corr undecided")
            rho = V(math.copysign(math.inf, corr.v))
    else:
        rho = corr / den
    ip = [S[6 + k] - imf * S[9 + k] for k in range(3)]
    tp = [S[12 + k] - tmf * S[9 + k] for k in range(3)]
    ipf, tpf = [p.f32(x) for x in ip], [p.f32(x) for x in tp]
    iph = [p.f32(Hi[a][0] * ipf[0] + Hi[a][1] * ipf[1] + Hi[a][2] * ipf[2]) for a in range(3)]
    lam_n = inorm * inorm - (ipf[0] * iph[0] + ipf[1] * iph[1] + ipf[2] * iph[2])
    lam_d = corr - (tpf[0] * iph[0] + tpf[1] * iph[1] + tpf[2] * iph[2])
    if p.test(lam_d.hi() <= 0.0, lam_d.lo() <= 0.0):
        return Mf, E.FAILED_LAMBDA, rho
    if math.isnan(rho.v):
        return Mf, E.FAILED_NAN, rho
    lam = lam_n / lam_d
    ep = [p.f32(lam * tp[k] - ip[k]) for k in range(3)]
    dp = [p.f32(Hi[a][0] * ep[0] + Hi[a][1] * ep[1] + Hi[a][2] * ep[2]) for a in range(3)]
    a10 = p.fn(math.asin, 1.0 / math.sqrt(max(1.0 - Mf[3] * Mf[3], 1e-300)), V(Mf[3]), ulps)
    theta = dp[0] + a10
    m02 = float(np.float32(Mf[2]) + np.float32(dp[1].v))
    m12 = float(np.float32(Mf[5]) + np.float32(dp[2].v))
    co = p.f32(p.fn(math.cos, min(1.0, abs(math.sin(theta.v)) + theta.r), theta, ulps)).v
    si = p.f32(p.fn(math.sin, min(1.0, abs(math.cos(theta.v)) + theta.r), theta, ulps)).v
    M2 = (co, -si, m02, si, co, m12)
    x = rho - last
    lo = 0.0 if x.lo() <= 0.0 <= x.hi() else min(abs(x.lo()), abs(x.hi()))
    hi = max(abs(x.lo()), abs(x.hi()))
    conv = p.test(hi < eps, lo < eps)
    return M2, (E.CONVERGED if conv else CONTINUE), rho


def bits(M):
    """float32 bit patterns of a map given as six values or a (2, 3) array."""
    return tuple(int(b) for b in np.asarray(M, np.float32).reshape(6).view(np.uint32))


class StepSet:
    """What one iteration can produce: ``outcomes`` {(map bits, flag)}, the rho interval [rho_lo, rho_hi], the fork count and the
    largest bound / |value| ratio at the sums (for reporting)."""

    def __init__(self, outcomes, rho_lo, rho_hi, forks):
        self.outcomes, self.rho_lo, self.rho_hi, self.forks = outcomes, rho_lo, rho_hi, forks

    def contains(self, M, flag, rho=None):
        if (bits(M), flag) not in self.outcomes:
            return False
        if rho is None:
            return True
        if math.isnan(self.rho_lo):
            return math.isnan(rho)
        return self.rho_lo <= rho <= self.rho_hi

    def maps(self):
        return sorted({m for m, _ in self.outcomes})


def step_from_sums(S, R, M, last, eps=1e-5, ulps=ULP_DEVICE + ULP_HOST):
    """Every outcome of one kernel iteration from sums S (with bounds R) and the float32 map M it starts from."""
    Mf = tuple(float(x) for x in np.asarray(M, np.float32).reshape(6))
    sv = [V(s, r) for s, r in zip(S, R)]
    outcomes, rlo, rhi = set(), math.inf, -math.inf
    choices, leaves = [], 0
    while True:
        p = _Path(choices)
        M2, fl, rho = _step(p, sv, Mf, V(last), eps, ulps)
        leaves += 1
        if leaves - 1 > MAX_FORKS:
            raise BoundTooLoose("more than %d forks in one iteration" % MAX_FORKS)
        outcomes.add((bits(M2), fl))
        if math.isnan(rho.v):
            rlo = rhi = math.nan
        elif not math.isnan(rlo):
            rlo, rhi = min(rlo, rho.lo()), max(rhi, rho.hi())
        choices = p.choices
        i = len(choices) - 1
        while i >= 0 and choices[i] + 1 >= p.widths[i]:
            i -= 1
        if i < 0:
            break
        choices = choices[:i] + [choices[i] + 1]
    return StepSet(outcomes, rlo, rhi, leaves - 1)


def step_set(tmpl, img, M, last, eps=1e-5, cluster=8, device=True):
    """Every outcome of one kernel iteration on (template, current plane) from the float32 map M, with ``last`` the rho the
    previous iteration reported (-1 before the first).  ``cluster``: CTAs per sequence (8 on the GPU, 1 in the simulator);
    ``device``: the kernel's cos / sin / asin are CUDA's (else the host's libm)."""
    S, R = sums_with_bound(tmpl, img, M, cluster)
    st = step_from_sums(S, R, M, last, eps, (ULP_DEVICE + ULP_HOST) if device else 2 * ULP_HOST)
    st.sum_ratio = max((r / abs(s) if s else 0.0) for s, r in zip(S, R))
    return st


def oracle_sums(sm):
    """oracle/ecc.py ``sums`` as the kernel's 21-vector."""
    J = sm["SJJ"]
    return ([sm["n"], sm["SI"], sm["SII"], sm["ST"], sm["STT"], sm["STI"]] + list(sm["SJI"]) + list(sm["SJ"]) + list(sm["SJT"])
            + [J[0, 0], J[0, 1], J[0, 2], J[1, 1], J[1, 2], J[2, 2]])
