"""TEST INFRASTRUCTURE: extended-precision reference, with a running error bound, of the tracker's Kalman and IoU arithmetic:
csrc/b2t_kalman.cuh (kf_q, kf_r, kf_predict, kf_update, kf_initiate, kf_gmc, det_to_meas, mean_to_tlwh / mean_to_tlbr) and the
kalman_gating_kernel / iou_cost_kernel of csrc/b2t_tracker.cu.  Shared by the GPU tier (tests/test_gpu_kalman_bounds.py) and the
CPU tier (tests/test_hostsim_kalman_bounds.py).

Every function below restates the kernel in the kernel's own operation order, on the exact values the kernel read.  A value is a
``B``: the reference value ``v`` (np.longdouble, 64-bit significand), a first-order running bound ``e`` on |kernel - v|, and the
magnitude ``m`` (the same expression evaluated on absolute values, the scale a rounding error is measured against).  With u the unit
roundoff of the kernel's type T (2^-24 for float, 2^-53 for double) plus the reference's own 2^-64, and r the rounded result:
  * a + b, a - b :  ea + eb + u|r|
  * a * b        :  |a| eb + |b| ea + ea eb + u|r|
  * a / b        :  (ea + |r| eb) / (|b| - eb) + u|r|         (the reciprocal is 1 / b)
  * sqrt(a)      :  ea / (sqrt(a) + sqrt(a - ea)) + u|r|       (<= ea / (2 sqrt(a - ea)))
The kernel is built with --fmad=false and IEEE division and square root, so each of its operations is rounded once and the rules
hold term by term -- and an operation whose operands are all exact (bound 0: inputs, constants, results of such operations) is
evaluated exactly as the kernel does it, in its type, with bound 0.  The places where the reference itself rounds to float32 (noise_std / noise_var with mean_f32, NSA's (1 - conf),
the float32 box arithmetic of basetrack.py) are part of the function being computed: they are evaluated by rounding the reference
value to float32, and contribute 2 u32 |x| of their own only when their input already carries an error (two inputs within e of
each other round to float32 values at most e + 2 u32 |x| apart).  det_to_meas reads float32 inputs and is evaluated exactly.

Slack for what the first-order rules leave out (products of two bounds inside sqrt, the reference's final rounding to compare):
  bound = 1.01 e + ulp_T(|v|)
The check is |got - v| <= bound per element.  ``cap_ok`` asserts the bound is not vacuous: on well-conditioned inputs every bound
stays below 2^-12 of its magnitude m."""
import numpy as np

LD = np.longdouble
U32 = 2.0 ** -24
U64 = 2.0 ** -53
U_REF = float(np.finfo(np.longdouble).eps) / 2
SLACK = 1.01
CAP = 2.0 ** -12

FMT_XYAH, FMT_XYWH, FMT_NSA = 0, 1, 2


def unit(f32):
    return (U32 if f32 else U64) + U_REF


def _a(x):
    return np.abs(np.asarray(x, np.float64))


def _exact(a, b, r, e, u, fn):
    """Where every operand is exact (bound 0) the kernel's result is one IEEE operation on known values: evaluate it exactly in
    the kernel's type (float32 for u >= 2^-24, else float64), bound 0."""
    x = (a.e == 0) if b is None else ((a.e == 0) & (b.e == 0))
    if not np.any(x):
        return r, e
    dt = np.float32 if u > 1e-12 else np.float64
    with np.errstate(all="ignore"):
        rx = (fn(a.v.astype(dt)) if b is None else fn(a.v.astype(dt), b.v.astype(dt))).astype(LD)
    return np.where(x, rx, r), np.where(x, 0.0, e)


class B:
    """A reference value with its running error bound and magnitude; arrays broadcast (one entry per track / measurement).
    ``ei`` is the same first-order bound without the exact evaluation of exact-operand operations: the rounding a different
    evaluation order of the same operations (the oracle's NumPy / LAPACK) may commit."""
    __slots__ = ("v", "e", "m", "u", "ei")

    def __init__(self, v, u, e=None, m=None, ei=None):
        self.v = np.asarray(v, LD)
        self.u = u
        self.e = np.zeros(self.v.shape) if e is None else np.broadcast_to(np.asarray(e, np.float64), self.v.shape).copy()
        self.m = _a(self.v) if m is None else np.broadcast_to(np.asarray(m, np.float64), self.v.shape).copy()
        self.ei = self.e.copy() if ei is None else np.broadcast_to(np.asarray(ei, np.float64), self.v.shape).copy()

    def _lift(self, o):
        return o if isinstance(o, B) else B(o, self.u)

    def add(self, o, u=None):
        o = self._lift(o)
        uu = u or self.u
        r = self.v + o.v
        ei = self.ei + o.ei + uu * _a(r)
        r, e = _exact(self, o, r, self.e + o.e + uu * _a(r), uu, np.add)
        return B(r, self.u, e, self.m + o.m, ei)

    def sub(self, o, u=None):
        o = self._lift(o)
        uu = u or self.u
        r = self.v - o.v
        ei = self.ei + o.ei + uu * _a(r)
        r, e = _exact(self, o, r, self.e + o.e + uu * _a(r), uu, np.subtract)
        return B(r, self.u, e, self.m + o.m, ei)

    def mul(self, o, u=None):
        o = self._lift(o)
        uu = u or self.u
        r = self.v * o.v
        ei = _a(self.v) * o.ei + _a(o.v) * self.ei + self.ei * o.ei + uu * _a(r)
        r, e = _exact(self, o, r, _a(self.v) * o.e + _a(o.v) * self.e + self.e * o.e + uu * _a(r), uu, np.multiply)
        return B(r, self.u, e, self.m * o.m, ei)

    def div(self, o, u=None):
        o = self._lift(o)
        uu = u or self.u
        with np.errstate(divide="ignore", invalid="ignore", over="ignore"):
            r = self.v / o.v

            def rule(ea, eb):
                den = _a(o.v) - eb
                return np.where(den > 0, (ea + _a(r) * eb) / np.where(den > 0, den, 1.0), np.inf) + uu * _a(r)
            e, ei = rule(self.e, o.e), rule(self.ei, o.ei)
            m = self.m / _a(o.v)
        r, e = _exact(self, o, r, e, uu, np.divide)
        return B(r, self.u, e, m, ei)

    def sqrt(self):
        with np.errstate(invalid="ignore", divide="ignore"):
            r = np.sqrt(self.v)

            def rule(ea):
                lo = np.sqrt(np.maximum(self.v.astype(np.float64) - ea, 0.0))
                return np.where(ea > 0, ea / (_a(r) + lo), 0.0) + self.u * _a(r)
            e, ei = rule(self.e), rule(self.ei)
        r, e = _exact(self, None, r, e, self.u, np.sqrt)
        return B(r, self.u, e, np.sqrt(self.m), ei)

    __add__, __sub__, __mul__, __truediv__ = add, sub, mul, div

    def r32(self):
        """The reference's own rounding to float32 (a quirk of its dtype, not an error of the kernel)."""
        r = self.v.astype(np.float32).astype(LD)
        grow = lambda ea: np.where(ea > 0, ea + 2 * U32 * (_a(self.v) + ea), 0.0)    # noqa: E731
        return B(r, self.u, grow(self.e), self.m, grow(self.ei))

    def take(self, i):
        """the entries at index array i (first axis)"""
        return B(self.v[i], self.u, self.e[i], self.m[i], self.ei[i])

    def where(self, mask, o):
        o = self._lift(o)
        return B(np.where(mask, self.v, o.v), self.u, np.where(mask, self.e, o.e), np.where(mask, self.m, o.m), np.where(mask, self.ei, o.ei))


def const(x, f32, u):
    """A constant as the kernel holds it: (T)x."""
    return B(np.float32(x) if f32 else np.float64(x), u)


def inputs(a, f32):
    """Exact kernel inputs (float32 or float64 array) -> B."""
    return B(np.asarray(a, np.float32 if f32 else np.float64), unit(f32))


# ---------------------------------------------------------------- b2t_kalman.cuh
def noise_std(weight, base, f32_quirk, f32):
    """b2t_kalman.cuh:41-44.  weight: a Python float constant of the kernel ((T)(1.0/20) ...), base: B."""
    if f32:
        return const(weight, True, base.u).mul(base)
    if f32_quirk:
        w = np.float32(np.float64(weight))
        return base.r32().mul(B(w, base.u), u=U32 + U_REF)
    return const(weight, False, base.u).mul(base)


def noise_var(s, f32_quirk, f32):
    """b2t_kalman.cuh:46-49."""
    if f32:
        return s.mul(s)
    if f32_quirk:
        f = s.r32()
        return f.mul(f, u=U32 + U_REF)
    return s.mul(s)


def kf_q(r, fmt, w, h, q_f32, f32):
    """b2t_kalman.cuh:52-66.  Process noise Q[r][r]."""
    pos = r < 4
    rr = r & 3
    wgt = 1.0 / 20 if pos else 1.0 / 160
    if fmt == FMT_XYWH:
        s = noise_std(wgt, h if rr & 1 else w, q_f32, f32)
    elif rr == 2:
        c = 1e-2 if pos else 1e-5
        s = B(np.broadcast_to(np.float32(c) if (f32 or q_f32) else np.float64(c), h.v.shape), h.u)
    else:
        s = noise_std(wgt, h, q_f32, f32)
    return noise_var(s, q_f32, f32)


def kf_r(c, fmt, w, h, mean_f32, conf, f32):
    """b2t_kalman.cuh:94-112.  Measurement noise R[c][c]; conf: None (no confidence) or a float32 array (one per track)."""
    u = h.u
    if fmt == FMT_XYWH:
        s = noise_std(1.0 / 20, h if c & 1 else w, mean_f32, f32)
        return noise_var(s, mean_f32, f32)
    s = B(np.broadcast_to(np.float32(0.1) if f32 else np.float64(0.1), h.v.shape), u) if c == 2 else noise_std(1.0 / 20, h, mean_f32, f32)
    if fmt == FMT_NSA and conf is not None:
        cf = np.asarray(conf, np.float32)
        omc = B(np.float32(1) - cf, u)                                   # float32 subtraction, evaluated exactly as the kernel does
        if f32:
            return noise_var(omc.mul(s), True, True)
        if c == 2:
            s2 = B((np.float32(1) - cf) * np.float32(0.1), u)            # float32 * float32 constant, exact emulation
            return noise_var(s2, mean_f32, False)
        if mean_f32:
            return noise_var(omc.mul(s.r32(), u=U32 + U_REF), True, False)
        s = omc.mul(s)
    return noise_var(s, False, f32)


def kf_r_mixed(c, fmt, w, h, mean_f32, conf, f32):
    """kf_r with a per-track mean_f32 mask (the kernel's flag bit)."""
    mf = np.asarray(mean_f32, bool)
    if f32 or not mf.any():
        return kf_r(c, fmt, w, h, False, conf, f32)
    if mf.all():
        return kf_r(c, fmt, w, h, True, conf, f32)
    return kf_r(c, fmt, w, h, True, conf, f32).where(mf, kf_r(c, fmt, w, h, False, conf, f32))


def state(mean, cov, f32):
    """(n, 8), (n, 8, 8) kernel inputs -> (list of 8 B, 8 x 8 nested list of B)."""
    mean = np.asarray(mean)
    cov = np.asarray(cov)
    m = [inputs(mean[:, r], f32) for r in range(8)]
    P = [[inputs(cov[:, r, j], f32) for j in range(8)] for r in range(8)]
    return m, P


def kf_predict(m, P, fmt, zero_vh, q_f32, f32):
    """b2t_kalman.cuh:71-90.  zero_vh: per-track bool array (FLAG_NOT_TRACKED)."""
    m = list(m)
    m[7] = m[7].where(~np.asarray(zero_vh, bool), 0.0)
    w, h = m[2], m[3]
    lrow = [[P[r][j] + P[r + 4][j] if r < 4 else P[r][j] for j in range(8)] for r in range(8)]
    nm = [m[r] + m[r + 4] if r < 4 else m[r] for r in range(8)]
    nP = []
    for r in range(8):
        q = kf_q(r, fmt, w, h, q_f32, f32)
        row = []
        for j in range(8):
            v = lrow[r][j] + lrow[r][(j + 4) & 7] if j < 4 else lrow[r][j]
            if j == r:
                v = v + q
            row.append(v)
        nP.append(row)
    return nm, nP


def innovation_cov(m, P, fmt, mean_f32, conf, f32):
    """S = P[:4, :4] + diag(R), as kf_update (b2t_kalman.cuh:118-125) and kalman_project_kernel (b2t_tracker.cu:107-114) form it."""
    S = [[P[a][b] for b in range(4)] for a in range(4)]
    for c in range(4):
        S[c][c] = S[c][c] + kf_r_mixed(c, fmt, m[2], m[3], mean_f32, conf, f32)
    return S


def kf_update(m, P, fmt, z, mean_f32, conf, f32):
    """b2t_kalman.cuh:117-168.  z: list of 4 B (the measurement the kernel read)."""
    S = innovation_cov(m, P, fmt, mean_f32, conf, f32)
    one = const(1.0, f32, m[0].u)
    L = [[None] * 4 for _ in range(4)]
    inv = [None] * 4
    L[0][0] = S[0][0].sqrt(); inv[0] = one / L[0][0]
    L[1][0] = S[1][0] * inv[0]
    L[2][0] = S[2][0] * inv[0]
    L[3][0] = S[3][0] * inv[0]
    L[1][1] = (S[1][1] - L[1][0] * L[1][0]).sqrt(); inv[1] = one / L[1][1]
    L[2][1] = (S[2][1] - L[2][0] * L[1][0]) * inv[1]
    L[3][1] = (S[3][1] - L[3][0] * L[1][0]) * inv[1]
    L[2][2] = ((S[2][2] - L[2][0] * L[2][0]) - L[2][1] * L[2][1]).sqrt(); inv[2] = one / L[2][2]
    L[3][2] = ((S[3][2] - L[3][0] * L[2][0]) - L[3][1] * L[2][1]) * inv[2]
    L[3][3] = (((S[3][3] - L[3][0] * L[3][0]) - L[3][1] * L[3][1]) - L[3][2] * L[3][2]).sqrt(); inv[3] = one / L[3][3]
    G = []
    for r in range(8):                                                   # gain row r (b2t_kalman.cuh:140-148)
        p = P[r]
        g = [None] * 4
        g[0] = p[0] * inv[0]
        g[1] = (p[1] - L[1][0] * g[0]) * inv[1]
        g[2] = ((p[2] - L[2][0] * g[0]) - L[2][1] * g[1]) * inv[2]
        g[3] = (((p[3] - L[3][0] * g[0]) - L[3][1] * g[1]) - L[3][2] * g[2]) * inv[3]
        g[3] = g[3] * inv[3]
        g[2] = (g[2] - L[3][2] * g[3]) * inv[2]
        g[1] = ((g[1] - L[2][1] * g[2]) - L[3][1] * g[3]) * inv[1]
        g[0] = (((g[0] - L[1][0] * g[1]) - L[2][0] * g[2]) - L[3][0] * g[3]) * inv[0]
        G.append(g)
    inn = [z[c] - m[c] for c in range(4)]                                # b2t_kalman.cuh:150-156
    nm = []
    for r in range(8):
        acc = inn[0] * G[r][0]
        for c in range(1, 4):
            acc = acc + inn[c] * G[r][c]
        nm.append(m[r] + acc)
    skt = [[((S[a][0] * G[r][0] + S[a][1] * G[r][1]) + S[a][2] * G[r][2]) + S[a][3] * G[r][3] for a in range(4)] for r in range(8)]
    nP = []
    for r in range(8):                                                   # b2t_kalman.cuh:161-167
        row = []
        for j in range(8):
            d = G[r][0] * skt[j][0]
            for a in range(1, 4):
                d = d + G[r][a] * skt[j][a]
            row.append(P[r][j] - d)
        nP.append(row)
    return nm, nP


def kf_initiate(z, fmt, f32):
    """b2t_kalman.cuh:171-188.  z: (k, 4) kernel input (float32-representable values in either dtype)."""
    z = np.asarray(z)
    u = unit(f32)
    zb = [inputs(z[:, q], f32) for q in range(4)]
    k = len(z)
    m = [zb[r] if r < 4 else B(np.zeros(k), u) for r in range(8)]
    diag = []
    for r in range(8):
        pos = r < 4
        rr = r & 3
        if fmt == FMT_XYWH:
            base = zb[3] if rr & 1 else zb[2]
            s = base.r32().mul(B(np.float32(0.1 if pos else 0.0625), u), u=U32 + U_REF)
            var = s.mul(s, u=U32 + U_REF)
        elif rr == 2:
            c = 1e-2 if pos else 1e-5
            var = B(np.full(k, np.float32(c)), u).mul(B(np.float32(c), u)) if f32 else B(np.full(k, c), u).mul(B(c, u))
        else:
            s = zb[3].r32().mul(B(np.float32(0.1 if pos else 0.0625), u), u=U32 + U_REF)
            var = s.mul(s)                                              # float32 std squared in T
        diag.append(var)
    P = [[diag[r] if j == r else B(np.zeros(k), u) for j in range(8)] for r in range(8)]
    return m, P


def kf_gmc(m, P, warp6):
    """b2t_kalman.cuh:192-215.  warp6: the six values {a00, a01, tx, a10, a11, ty} as the kernel holds them (T)."""
    u = m[0].u
    w = [B(x, u) for x in warp6]
    nm = []
    mrow = []
    for r in range(8):
        odd = r & 1
        ra, rb = (w[3], w[4]) if odd else (w[0], w[1])
        e0, o0 = r & 6, (r & 6) | 1
        v = ra * m[e0] + rb * m[o0]
        if r == 0:
            v = v + w[2]
        if r == 1:
            v = v + w[5]
        nm.append(v)
        mrow.append([ra * P[e0][j] + rb * P[o0][j] for j in range(8)])
    nP = []
    for r in range(8):
        row = []
        for j in range(8):
            ca, cb = (w[3], w[4]) if j & 1 else (w[0], w[1])
            row.append(mrow[r][j & 6] * ca + mrow[r][(j & 6) | 1] * cb)
        nP.append(row)
    return nm, nP


def det_to_meas(fmt, tlbr):
    """b2t_kalman.cuh:219-232: float32 arithmetic in either build, evaluated exactly.  tlbr (k, 4) float32 -> (k, 4) float32."""
    x1, y1, x2, y2 = [np.asarray(tlbr, np.float32)[:, q] for q in range(4)]
    w, h = x2 - x1, y2 - y1
    two = np.float32(2)
    if fmt == FMT_XYWH:
        return np.stack([x1 + np.floor(w / two), y1 + np.floor(h / two), w, h], 1).astype(np.float32)
    return np.stack([x1 + w / two, y1 + h / two, w / h, h], 1).astype(np.float32)


def mean_to_tlwh(fmt, m, mean_f32, f32):
    """b2t_kalman.cuh:235-251.  m: list of >= 4 B; mean_f32: per-track bool mask (flag bit 1 of the slot)."""
    def path(q):
        if q and not f32:
            w, h = m[2].r32(), m[3].r32()
            uu = U32 + U_REF
            if fmt != FMT_XYWH:
                w = w.mul(h, u=uu)
            return [m[0].r32().sub(w.div(2.0, u=uu), u=uu), m[1].r32().sub(h.div(2.0, u=uu), u=uu), w, h]
        w, h = m[2], m[3]
        if fmt != FMT_XYWH:
            w = w * h
        return [m[0] - w / 2.0, m[1] - h / 2.0, w, h]
    mf = np.asarray(mean_f32, bool)
    if f32 or not mf.any():
        return path(False)
    if mf.all():
        return path(True)
    a, b = path(True), path(False)
    return [x.where(mf, y) for x, y in zip(a, b)]


# ---------------------------------------------------------------- b2t_tracker.cu
def gating(fmt, mean, cov, meas, only_position, metric, f32, mean_f32=False):
    """kalman_gating_kernel (b2t_tracker.cu:117-150): one state (mean (8,), cov (8, 8)) against meas (m, 4) -> B of (m,)."""
    mm = len(meas)
    u = unit(f32)
    dt = np.float32 if f32 else np.float64
    mean = np.asarray(mean, dt)
    cov = np.asarray(cov, dt)
    meas = np.asarray(meas, dt)
    mb = [B(np.full(mm, mean[a]), u) for a in range(4)]
    nd = 2 if only_position else 4
    S = [[B(np.full(mm, cov[a, b]), u) for b in range(4)] for a in range(4)]
    d = []
    for a in range(4):
        S[a][a] = S[a][a] + kf_r(a, fmt, B(np.full(mm, mean[2]), u), B(np.full(mm, mean[3]), u), mean_f32, None, f32)
        d.append(B(meas[:, a], u) - mb[a])
    acc = B(np.zeros(mm), u)
    if metric == 1:
        for a in range(nd):
            acc = acc + d[a] * d[a]
        return acc
    L = [[None] * 4 for _ in range(4)]
    for a in range(nd):
        for b in range(a + 1):
            s = S[a][b]
            for q in range(b):
                s = s - L[a][q] * L[b][q]
            L[a][b] = s.sqrt() if a == b else s / L[b][b]
    for a in range(nd):
        s = d[a]
        for q in range(a):
            s = s - L[a][q] * d[q]
        d[a] = s / L[a][a]
        acc = acc + d[a] * d[a]
    return acc


def iou_plus1(a, b, f32):
    """b2t_iou.cuh:14-24 for every pair: a (n, 4), b (m, 4) tlbr -> (IoU B of (n, m), ambiguous mask).  A pair whose iw or ih
    lies within its bound of 0 may take either branch of the kernel's `> 0` test: it is reported as ambiguous."""
    u = unit(f32)
    dt = np.float32 if f32 else np.float64
    a = np.asarray(a, dt)[:, None, :]
    b = np.asarray(b, dt)[None, :, :]
    one = const(1.0, f32, u)
    iw = B(np.minimum(a[..., 2], b[..., 2]), u) - B(np.maximum(a[..., 0], b[..., 0]), u) + one
    ih = B(np.minimum(a[..., 3], b[..., 3]), u) - B(np.maximum(a[..., 1], b[..., 1]), u) + one
    area_a = (B(a[..., 2], u) - B(a[..., 0], u) + one) * (B(a[..., 3], u) - B(a[..., 1], u) + one)
    area_b = (B(b[..., 2], u) - B(b[..., 0], u) + one) * (B(b[..., 3], u) - B(b[..., 1], u) + one)
    inter = iw * ih
    ua = (area_a + area_b) - inter
    iou = inter / ua
    zero = ~((iw.v > 0) & (ih.v > 0))
    amb = (_a(iw.v) <= iw.e) | (_a(ih.v) <= ih.e)
    return B(np.where(zero, 0, iou.v), u, np.where(zero, 0, iou.e), np.where(zero, 0, iou.m)), amb


# ---------------------------------------------------------------- the check
def ulp(v, f32):
    a = _a(v)
    info = np.finfo(np.float32 if f32 else np.float64)
    return np.spacing(np.maximum(a, float(info.tiny)).astype(np.float32 if f32 else np.float64)).astype(np.float64)


def bound(ref, f32):
    return SLACK * ref.e + ulp(ref.v.astype(np.float64), f32)


def bound_any_order(ref, f32):
    """the bound of an evaluation of the same operations in another order (no exact shortcuts)"""
    return SLACK * ref.ei + ulp(ref.v.astype(np.float64), f32)


def check(got, ref, f32, what):
    """|got - ref.v| <= bound elementwise; every value finite.  Returns the largest err / bound."""
    got = np.asarray(got, np.float64)
    v = np.broadcast_to(ref.v, got.shape)
    assert np.isfinite(got).all(), "%s: non-finite output at %s" % (what, np.argwhere(~np.isfinite(got))[0])
    b = np.broadcast_to(bound(ref, f32), got.shape)
    assert np.isfinite(b).all(), "%s: the reference bound is not finite at %s" % (what, np.argwhere(~np.isfinite(b))[0])
    err = np.abs(got.astype(LD) - v).astype(np.float64)
    bad = err > b
    if bad.any():
        i = tuple(np.argwhere(bad)[0])
        raise AssertionError("%s: %d of %d values beyond the bound, worst err/bound %.3g; first at %s: got %r ref %r bound %.3g" % (
            what, int(bad.sum()), bad.size, float((err / b).max()), i, float(got[i]), float(v[i]), float(b[i])))
    return float((err / b).max()) if err.size else 0.0


def cap_ok(ref, f32, what, cap=CAP):
    """The bound is not vacuous: below cap times the magnitude of every output."""
    pos = ref.m > 0
    assert (ref.e[~pos] == 0).all(), "%s: an exact zero carries an error bound" % what
    r = bound(ref, f32)[pos] / ref.m[pos]
    assert (r <= cap).all(), "%s: bound / magnitude %.3g above the cap %.3g" % (what, float(r.max()), cap)
    return float(r.max()) if r.size else 0.0


def stack(bs):
    """list of B of shape (n,) -> B of shape (n, len)."""
    return B(np.stack([b.v for b in bs], -1), bs[0].u, np.stack([b.e for b in bs], -1), np.stack([b.m for b in bs], -1),
             np.stack([b.ei for b in bs], -1))


def stack_cov(P):
    """8 x 8 (or 4 x 4) nested list of B of shape (n,) -> B of shape (n, 8, 8)."""
    rows = [stack(row) for row in P]
    return B(np.stack([r.v for r in rows], -2), rows[0].u, np.stack([r.e for r in rows], -2), np.stack([r.m for r in rows], -2),
             np.stack([r.ei for r in rows], -2))
