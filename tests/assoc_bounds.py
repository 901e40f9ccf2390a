"""TEST INFRASTRUCTURE: every association of the fused step certified, frame by frame from the tracker's own stored state, as an
optimal thresholded assignment for costs within a derived float64 interval -- the association-side counterpart of tests/step_bounds.py,
shared by the GPU tier (tests/test_gpu_step_assoc.py) and the CPU tier (tests/test_hostsim_step_assoc.py).

step_bounds.check_stream hands each frame (its on_frame callback) the before-state in list order, each slot's predicted or warped
state with its bound, the float32-mean flag the association read, the detection each slot was updated with and the stat words.  From
that alone (nothing is read back) the certifier restates which rows, columns and threshold each association uses
(b2t_step.cuh track_step_cta; oracle/trackers.py:259-293, tests/reid_track_oracle.py:98-128, tests/strongsort_oracle.py:86-122,
tests/uavmot_oracle.py:183-225):
  * high / low rows in float32 (score >= det_thresh, low_thresh < score < det_thresh; SORT and StrongSORT: score > det_thresh, no low
    rows), boxes with a non-finite coordinate or no height (or, xywh, no width) in neither;
  * association 1: pool (activated tracked ++ lost, list order) x high rows at t1 (0.9; SORT iou_thresh; StrongSORT, UAVMOT 0.7);
  * association 2: association 1's leftover pool rows -- only the Tracked ones for ByteTrack, StrongSORT and UAVMOT (q4, q18) -- x
    the low rows, or for StrongSORT (kChain) x association 1's leftover high rows, IoU at 0.5;
  * association 3: unconfirmed x association 1's leftover high rows (StrongSORT: association 2's), at t3 (0.7; SORT iou_thresh + 0.1);
  * UAVMOT (q20): the IoU solve at 0.7 decides only whether the fused solve at 0.8 runs -- it does when that solve matched some pair
    other than (0, 0); the fused solve's matching then replaces it.
Every entry is an interval [L, U] that contains the kernel's cost:
  * "+1" IoU distance (b2t_iou.cuh) on the row box mean_to_tlbr of the predicted mean +- its kalman_ref bound, each operation's rounding
    in the build's T added by tests/kalman_ref.py's rules; a pair whose iw or ih lies within its bound of 0 may take either branch
    (distance 1 or the quotient) and gets the hull of both;
  * BoT-SORT with ReID, App = 0.5 (1 - a.b / (|a| |b|)) (app_costs): a.b, a.a, b.b in float64 from the float32 rows, plus the kernel's
    accumulation in T -- each lane sums D / 128 float4 chunks, 4 products and 3 additions per chunk, then 5 shuffle levels, so each
    product passes through at most 1 + 3 + D / 128 + 5 roundings: gamma_k sum |a_i b_i|.  App > theta_emb becomes 1, the cost is
    min(IoU distance, App) where the IoU distance is <= theta_iou; an interval that straddles a gate takes the hull of both outcomes;
  * StrongSORT, gamma IoU distance + (1 - gamma) Euclidean distance (build_csr_dense), the distance and its bound from
    tests/featdist_ref.py, rounded to T in the float32 build;
  * UAVMOT, 0.98 IoU distance + (1 - 0.98) S, with S from tests/uavmot_oracle.structure_vectors on the predicted centres: every
    length comparison, arg max / arg min and truncated angle must stay decided under the centres' bound -- otherwise the check fails
    with "bound too loose".
Each update is assigned to an association by its row and column sets; a StrongSORT pool x high pair goes to association 1 when its
association-1 interval lies below t1, to association 2 when it lies at or above t1, and both splits are tried when it straddles t1.
The number of association-1 matches must equal stat word 11 (STAT_NMATCH0).  For each association with cost limit t the certificate
requires
  (a) every matched pair has L < t;
  (b) the kernel's lapjv objective sum_matched L + (unmatched rows + unmatched columns) t / 2 is at most the best objective over the
      upper costs U (scipy's linear_sum_assignment on the extended matrix, tests/lap_ref.py / oracle/lapjv.py) -- necessary for the
      matching to be optimal for some cost matrix inside the intervals;
  (c) no unmatched row and unmatched column have U < t.
A failure names the association, frame, row slot, column detection and both intervals.  stats collects the largest interval width
of a matched or sub-threshold entry and the smallest slack of (b)."""
import itertools
import math

import numpy as np
from scipy.optimize import linear_sum_assignment

import featdist_ref as FR
import kalman_ref as R
import uavmot_oracle as UO
from oracle import kalman as K

T1 = dict(sort=None, bytetrack=0.9, botsort=0.9, strongsort=0.7, uavmot=0.7)
T3 = dict(sort=None, bytetrack=0.7, botsort=0.7, strongsort=0.7, uavmot=0.7)
T2, UAV_T1, UAV_LAMBDA = 0.5, 0.8, 0.98
MAX_SPLITS = 10           # StrongSORT pool x high pairs whose interval straddles t1: at most 2^10 splits are tried


class CertError(AssertionError):
    """a certificate failure (as opposed to an assertion of the frame-by-frame state check)"""


def _gamma(k, u):
    return k * u / (1 - k * u)


def _iv(b, f32):
    """(L, U) float64, rounded outwards, of a kalman_ref value and its bound"""
    bd = R.bound(b, f32)
    with np.errstate(invalid="ignore", over="ignore"):
        lo = (b.v - bd).astype(np.float64)
        hi = (b.v + bd).astype(np.float64)
    return np.nextafter(lo, -np.inf), np.nextafter(hi, np.inf)


def _lift(b, f32):
    """a kalman_ref value as a kernel input: the reference value with its whole bound as input error"""
    return R.B(b.v, b.u, R.bound(b, f32), b.m)


def _mn(a, b):
    return R.B(np.minimum(a.v, b.v), a.u, np.maximum(a.e, b.e), np.maximum(a.m, b.m))


def _mx(a, b):
    return R.B(np.maximum(a.v, b.v), a.u, np.maximum(a.e, b.e), np.maximum(a.m, b.m))


def row_boxes(base_mean, flags, fmt, f32):
    """the kernel's row boxes (fill_track_boxes: mean_to_tlbr with the slot's float32-mean flag) as 4 B of shape (n,)"""
    m = [_lift(x, f32) for x in base_mean[:4]]
    t = R.mean_to_tlwh(fmt, m, flags, f32)
    flags = np.asarray(flags, bool)
    plain = [t[0], t[1], t[2].add(t[0]), t[3].add(t[1])]
    if f32 or not flags.any():
        return plain
    u32 = R.U32 + R.U_REF
    narrow = [t[0], t[1], t[2].add(t[0], u=u32), t[3].add(t[1], u=u32)]
    return [a.where(flags, b) for a, b in zip(narrow, plain)]


def det_boxes(dets):
    """the kernel's column boxes: tlbr from the float32 tlwh (float32 arithmetic, exact here)"""
    tl = K.tlbr_to_tlwh_f32(np.asarray(dets, np.float32)[:, :4].reshape(-1, 4))
    tb = tl.copy()
    tb[:, 2:] += tb[:, :2]
    return tb


def iou_dist(rows, cols, f32):
    """(d, pos, amb): the IoU distance B of every (row, column) pair on the overlapping branch, the pairs that certainly take it, and
    the pairs whose iw or ih lies within its bound of 0 (either branch).  The others certainly cost exactly 1."""
    u = R.unit(f32)
    dt = np.float32 if f32 else np.float64
    a = [R.B(x.v[:, None], u, x.e[:, None], x.m[:, None]) for x in rows]
    c = np.asarray(cols, dt).reshape(-1, 4)
    b = [R.B(c[None, :, q], u) for q in range(4)]
    one = R.const(1.0, f32, u)
    with np.errstate(all="ignore"):
        iw = _mn(a[2], b[2]).sub(_mx(a[0], b[0])).add(one)
        ih = _mn(a[3], b[3]).sub(_mx(a[1], b[1])).add(one)
        area_a = a[2].sub(a[0]).add(one).mul(a[3].sub(a[1]).add(one))
        area_b = b[2].sub(b[0]).add(one).mul(b[3].sub(b[1]).add(one))
        inter = iw.mul(ih)
        d = one.sub(inter.div(area_a.add(area_b).sub(inter)))
    bw, bh = R.bound(iw, f32), R.bound(ih, f32)
    pos = (iw.v > bw) & (ih.v > bh)
    neg = (iw.v + bw <= 0) | (ih.v + bh <= 0)
    return d, pos, ~pos & ~neg


def _branch(pos, amb, on, off):
    """the interval of a cost whose IoU branch is `on` (an interval pair) where pos, exactly `off` where neither, the hull on amb"""
    lo = np.where(pos, on[0], off[0])
    hi = np.where(pos, on[1], off[1])
    lo = np.where(amb, np.minimum(on[0], off[0]), lo)
    hi = np.where(amb, np.maximum(on[1], off[1]), hi)
    return lo, hi


def iou_costs(rows, cols, f32):
    d, pos, amb = iou_dist(rows, cols, f32)
    L, U = _iv(d, f32)
    return _branch(pos, amb, (L, U), (np.ones_like(L), np.ones_like(U))), (d, pos, amb)


def reid_costs(rows, cols, tfeat, dfeat, f32, theta_iou, theta_emb):
    """min(IoU distance, App) with BoT-SORT's gates (app_costs, botsort.py:386-392)"""
    (Li, Ui), _ = iou_costs(rows, cols, f32)
    A = np.asarray(tfeat, np.float32).astype(np.float64).reshape(len(Li), -1)
    Bm = np.asarray(dfeat, np.float32).astype(np.float64).reshape(Li.shape[1], -1)
    D = A.shape[1]
    u = R.unit(f32)
    k = 1 + 3 + -(-D // 128) + 5
    g = _gamma(k, R.U32 if f32 else R.U64) + _gamma(D, R.U64)          # the kernel's accumulation + this float64 evaluation
    ab, sab = A @ Bm.T, np.abs(A) @ np.abs(Bm).T
    aa, bb = (A * A).sum(1)[:, None], (Bm * Bm).sum(1)[None, :]
    one = R.const(1.0, f32, u)
    with np.errstate(all="ignore"):
        cos = R.B(ab, u, g * sab).div(R.B(aa, u, g * aa).sqrt().mul(R.B(bb, u, g * bb).sqrt()))
        app = R.const(0.5, f32, u).mul(one.sub(cos))
    La, Ua = _iv(app, f32)
    dt = np.float32 if f32 else np.float64
    th_iou, th_emb = float(dt(theta_iou)), float(dt(theta_emb))
    La, Ua = np.where(La > th_emb, 1.0, La), np.where(Ua > th_emb, 1.0, Ua)     # App > theta_emb -> 1; a straddle spans [La, 1]
    fL, fU = np.minimum(La, Li), np.minimum(Ua, Ui)
    gate_in, gate_out = Ui <= th_iou, Li > th_iou
    lo = np.where(gate_in, fL, np.where(gate_out, Li, np.minimum(fL, Li)))
    hi = np.where(gate_in, fU, np.where(gate_out, Ui, np.maximum(fU, Ui)))
    return lo, hi


def strongsort_costs(rows, cols, tfeat, dfeat, f32, gamma):
    """gamma IoU distance + (1 - gamma) App (build_csr_dense), App = the feature distance of feat_dist_kernel rounded to T"""
    d, pos, amb = iou_dist(rows, cols, f32)
    u = R.unit(f32)
    D = np.asarray(tfeat).reshape(d.v.shape[0], -1).shape[1]
    ex = FR.exact(np.asarray(tfeat, np.float32).reshape(-1, D), np.asarray(dfeat, np.float32).reshape(-1, D))
    e = FR.bound(ex, D)
    if f32:
        e = e + R.U32 * (np.asarray(ex, np.float64) + e)
    app = R.B(ex, u, e)
    g, g1 = R.const(gamma, f32, u), R.const(1.0 - gamma, f32, u)
    one = R.B(np.ones(d.v.shape), u)
    with np.errstate(all="ignore"):
        on = _iv(g.mul(d).add(g1.mul(app)), f32)
        off = _iv(g.mul(one).add(g1.mul(app)), f32)
    return _branch(pos, amb, on, off)


# ---------------------------------------------------------------- UAVMOT's structure cost
def _track_structure(pts, dlt, tag):
    """structure vectors of the track points (n, 2) float64 whose kernel values lie within dlt (n,) of them (Euclidean): (sv (n, 3),
    err (n, 3)).  Every decision -- neighbour or not, which point is the farthest / nearest, the truncated directions -- must be the
    same for every point set inside the bound."""
    sv = UO.structure_vectors(pts, False)
    n = len(pts)
    err = np.zeros((n, 3))
    if n == 0:
        return sv, err
    Lm = UO.lengths(pts, False)
    for i in range(n):
        row = Lm[i]
        # |length - reference length| per neighbour; two exact points (bound 0) give the kernel the very operands, and the same length
        mg = dlt[i] + dlt + np.where((dlt[i] > 0) | (dlt > 0), 4 * R.U64 * np.maximum(row, 1.0), 0.0)
        others = np.arange(n) != i
        near = others & (mg > 0) & ((np.abs(row - UO.LOCAL_R) <= mg) | (row <= mg))
        if near.any():
            raise CertError("%s: UAVMOT structure of pool row %d: bound too loose (a length within %.3g of 0 or 400)" % (tag, i, mg[near].max()))
        nb = np.nonzero(others & (row < UO.LOCAL_R) & (row > 0))[0]
        if len(nb) == 0:
            continue
        lv = row[nb]
        jmax, jmin = nb[int(np.argmax(lv == lv.max()))], nb[int(np.argmax(lv == lv.min()))]
        for j, sgn in ((jmax, 1), (jmin, -1)):
            rest = nb[nb != j]
            gap = mg[j] + mg[rest]                      # exact points tie exactly as the kernel does: the first index wins both
            if len(rest) and ((sgn * (row[j] - row[rest]) <= gap) & (gap > 0)).any():
                raise CertError("%s: UAVMOT structure of pool row %d: bound too loose (the %s neighbour is not decided)" % (
                    tag, i, "farthest" if sgn > 0 else "nearest"))
        err[i, 0], err[i, 1] = mg[jmax], mg[jmin]
        if jmax != jmin:
            for j in (jmax, jmin):
                dx, dy = pts[j, 0] - pts[i, 0], pts[j, 1] - pts[i, 1]
                a = math.atan2(dy, dx) * 180 / math.pi
                m = math.degrees(math.asin(min(1.0, mg[j] / row[j]))) + 1e-9
                if mg[j] > 0 and abs(a - round(a)) <= m:
                    raise CertError("%s: UAVMOT structure of pool row %d: bound too loose (direction %.12g within %.3g of an integer)" % (
                        tag, i, a, m))
    return sv, err


def structure_cost_interval(sv_r, e_r, sv_c):
    """S = max(0, 1 - clip(u.v / (|u| |v|))) in float64 (uav_struct_dist) for rows with error e_r and exact columns"""
    u = R.unit(False)
    a = [R.B(sv_r[:, q][:, None], u, e_r[:, q][:, None]) for q in range(3)]
    b = [R.B(sv_c[:, q][None, :], u) for q in range(3)]
    with np.errstate(all="ignore"):
        nu = a[0].mul(a[0]).add(a[1].mul(a[1])).add(a[2].mul(a[2])).sqrt()
        nv = b[0].mul(b[0]).add(b[1].mul(b[1])).add(b[2].mul(b[2])).sqrt()
        c = a[0].mul(b[0]).add(a[1].mul(b[1])).add(a[2].mul(b[2])).div(nu.mul(nv))
    cl, cu = _iv(c, False)
    cl, cu = np.clip(cl, -1, 1), np.clip(cu, -1, 1)
    lo, hi = np.nextafter(1.0 - cu, -np.inf), np.nextafter(1.0 - cl, np.inf)
    return np.maximum(lo, 0.0), np.maximum(hi, 0.0)


def uavmot_costs(rows, cols, base_mean, pool_idx, hi_tlwh, tag):
    """0.98 IoU distance + (1 - 0.98) S (build_csr's StructCtx hook), float64"""
    d, pos, amb = iou_dist(rows, cols, False)
    pts = np.stack([base_mean[0].v[pool_idx].astype(np.float64), base_mean[1].v[pool_idx].astype(np.float64)], 1).reshape(-1, 2)
    exact = (base_mean[0].e[pool_idx] == 0) & (base_mean[1].e[pool_idx] == 0)      # evaluated exactly as the kernel does
    dlt = np.where(exact, 0.0, np.hypot(R.bound(base_mean[0], False)[pool_idx], R.bound(base_mean[1], False)[pool_idx]))
    sv_r, e_r = _track_structure(pts, dlt, tag)
    sv_c = UO.structure_vectors(UO.det_centres(hi_tlwh), True)
    Sl, Su = structure_cost_interval(sv_r, e_r, sv_c)
    u = R.unit(False)
    S = R.B((Sl.astype(np.longdouble) + Su) / 2, u, (Su - Sl) / 2 * 1.0000001)
    lam, lam1 = R.B(np.float64(UAV_LAMBDA), u), R.B(np.float64(1.0 - UAV_LAMBDA), u)
    one = R.B(np.ones(d.v.shape), u)
    with np.errstate(all="ignore"):
        on = _iv(lam.mul(d).add(lam1.mul(S)), False)
        off = _iv(lam.mul(one).add(lam1.mul(S)), False)
    return _branch(pos, amb, on, off)


# ---------------------------------------------------------------- the certificate
def certify(what, L, U, t, pairs, rows, cols, stats):
    """(a), (b), (c) for one association: L, U (n, m), threshold t, matched (row index, column index) pairs; rows / cols name the
    slots and detections for the report.  Returns nothing; raises CertError."""
    n, m = L.shape
    mr, mc = np.zeros(n, bool), np.zeros(m, bool)
    for i, j in pairs:
        if mr[i] or mc[j]:
            raise CertError("%s: row slot %d or column detection %d matched twice" % (what, rows[i], cols[j]))
        mr[i] = mc[j] = True
        if not L[i, j] < t:
            raise CertError("%s: (a) matched pair row slot %d, column detection %d has cost in [%.17g, %.17g], not below %g" % (
                what, rows[i], cols[j], L[i, j], U[i, j], t))
    if n and m:
        free = (~mr[:, None]) & (~mc[None, :]) & (U < t)
        if free.any():
            i, j = np.argwhere(free)[0]
            raise CertError("%s: (c) row slot %d and column detection %d are both unmatched with cost in [%.17g, %.17g] below %g" % (
                what, rows[i], cols[j], L[i, j], U[i, j], t))
        W = np.minimum(U - t, 0.0)
        r, c = linear_sum_assignment(W)
        terms = [float(x) for x in W[r, c]] + [t - float(L[i, j]) for i, j in pairs]
        slack = math.fsum(terms)
        tol = 8 * np.finfo(np.float64).eps * (math.fsum(abs(x) for x in terms) + 1e-300)
        if slack < -tol:
            kp = set(map(tuple, pairs))
            bp = [(int(i), int(j)) for i, j in zip(r, c) if W[i, j] < 0]
            diff = [p for p in kp.symmetric_difference(bp)][:4]
            raise CertError("%s: (b) the kernel's objective exceeds the best one over the upper costs by %.6g; pairs that differ: %s" % (
                what, -slack, ", ".join("slot %d - det %d [%.17g, %.17g]%s" % (rows[i], cols[j], L[i, j], U[i, j],
                                                                             " kernel" if (i, j) in kp else " best") for i, j in diff)))
        if pairs:
            stats["min_slack"] = min(stats.get("min_slack", np.inf), slack)
        live = (L < t)
        if live.any():
            w = (U - L)[live]
            stats["max_width"] = max(stats.get("max_width", 0.0), float(w.max()))
            rel = w / np.maximum(np.abs(U[live]), 1e-300)
            stats["max_rel_width"] = max(stats.get("max_rel_width", 0.0), float(rel.max()))
    stats["assoc"] = stats.get("assoc", 0) + 1
    stats["pairs"] = stats.get("pairs", 0) + len(pairs)


class Certifier:
    """on_frame callback of step_bounds.check_stream.  kind: sort / bytetrack / botsort / strongsort / uavmot; reid: BoT-SORT with
    appearance features."""

    def __init__(self, kind, fmt, f32, conf_thresh=0.2, iou_thresh=0.5, theta_iou=0.5, theta_emb=0.25, gamma=0.1, stats=None):
        self.kind, self.fmt, self.f32 = kind, fmt, f32
        self.conf, self.iou_thresh = conf_thresh, iou_thresh
        self.theta_iou, self.theta_emb, self.gamma = theta_iou, theta_emb, gamma
        self.stats = {} if stats is None else stats
        self.frames = 0
        self.edges = []             # stat word 15 per frame (association 1's candidate count)
        self.pools = []             # (pool rows, high rows) per frame

    # ---- the frame's row and column sets
    def _split(self, dets):
        sc = dets[:, 4]
        tl = K.tlbr_to_tlwh_f32(dets[:, :4]) if len(dets) else np.zeros((0, 4), np.float32)
        area = np.isfinite(dets[:, :4]).all(1) & (tl[:, 3] != 0)
        if self.fmt == K.FMT_XYWH:
            area &= tl[:, 2] != 0
        det_t = np.float32(self.conf)
        if self.kind in ("sort", "strongsort"):
            return np.nonzero((sc > det_t) & area)[0], np.zeros(0, np.int64)
        low_t = np.float32(self.conf - 0.3 if self.conf - 0.3 > 0.15 else 0.15)             # bytetrack.py:15
        him = sc >= det_t
        return np.nonzero(him & area)[0], np.nonzero(~him & (sc > low_t) & area)[0]

    def __call__(self, fr):
        self.frames += 1
        before, exist, tag = fr["before"], fr["exist"], fr["tag"]
        dets = np.asarray(fr["dets"], np.float32).reshape(-1, 6)
        hi, lo = self._split(dets)
        if fr["stat"] is not None:
            assert fr["stat"][4] == 0, "%s: STAT_ERR %d" % (tag, fr["stat"][4])
            self.edges.append(int(fr["stat"][15]))
            self.pools.append((int(fr["stat"][6]), int(fr["stat"][8])))
        if not exist:
            return
        idx = {s: k for k, s in enumerate(exist)}
        pool = [s for s in before if before[s]["pool"]]
        unconf = [s for s in before if not before[s]["pool"]]
        tracked0 = {s: before[s]["state"] == 1 for s in before}
        md = {s: int(fr["matched_det"][idx[s]]) for s in exist if fr["matched_det"][idx[s]] >= 0}
        base_mean = fr["base"][0]
        rb_all = row_boxes(base_mean, fr["uflag"], self.fmt, self.f32)
        colbox = det_boxes(dets) if len(dets) else np.zeros((0, 4), np.float32)
        self._ctx = dict(tag=tag, dets=dets, colbox=colbox, rb_all=rb_all, idx=idx, base_mean=base_mean, before=before,
                         feats=fr["feats"], hi=hi)
        his, los = set(hi.tolist()), set(lo.tolist())
        kind = self.kind
        t1 = self.iou_thresh if kind == "sort" else T1[kind]
        t3 = self.iou_thresh + 0.1 if kind == "sort" else T3[kind]

        # every update in its association
        up_pool = [(s, md[s]) for s in pool if s in md]
        up_unc = [(s, md[s]) for s in unconf if s in md]
        for s, d in up_pool:
            if d not in his and d not in los:
                raise CertError("%s: pool slot %d was updated by detection %d, which no association offers it" % (tag, s, d))
        for s, d in up_unc:
            if d not in his:
                raise CertError("%s: unconfirmed slot %d was updated by detection %d, which is not a high row" % (tag, s, d))
        pr = {s: k for k, s in enumerate(pool)}
        hc = {d: k for k, d in enumerate(hi.tolist())}

        C1 = self._costs("dense", pool, hi, t1) if kind == "strongsort" else None
        if kind == "strongsort":
            sure1 = [(s, d) for s, d in up_pool if C1[1][pr[s], hc[d]] < t1]
            sure2 = [(s, d) for s, d in up_pool if C1[0][pr[s], hc[d]] >= t1]
            amb = [p for p in up_pool if p not in sure1 and p not in sure2]
            if len(amb) > MAX_SPLITS:
                raise CertError("%s: bound too loose (%d association-1 / 2 pairs straddle t1)" % (tag, len(amb)))
            splits = [(sure1 + [p for p, b in zip(amb, bits) if b], sure2 + [p for p, b in zip(amb, bits) if not b])
                      for bits in itertools.product((True, False), repeat=len(amb))]
        else:
            splits = [([(s, d) for s, d in up_pool if d in his], [(s, d) for s, d in up_pool if d in los])]
        # A pool row that is neither Tracked nor Lost (a removed track still on the lost list) may be matched in association 1 without
        # an update (bytetrack.py:121-127: neither branch).  Such matches take detections all the same; their number is stat word 11
        # minus the visible ones, and every placement of them on the leftover high rows is tried.
        quiet = [s for s in pool if kind != "sort" and before[s]["state"] not in (1, 2)]
        first = None
        tried = 0
        for a1, a2 in splits:
            extra = [()]
            if quiet and fr["stat"] is not None:
                k = int(fr["stat"][11]) - len(a1)
                used = {d for _, d in a1}
                free = [d for d in hi.tolist() if d not in used]
                extra = [] if not 0 <= k <= len(quiet) else [
                    tuple(zip(rs, ds)) for rs in itertools.combinations(quiet, k) for ds in itertools.permutations(free, k)]
            for ex in extra:
                tried += 1
                if tried > 4096:
                    raise CertError("%s: bound too loose (more than 4096 association hypotheses)" % tag)
                try:
                    self._chain(fr, pool, unconf, hi, lo, tracked0, a1 + list(ex), a2, up_unc, C1, t1, t3)
                    return
                except CertError as e:
                    first = first or e
        raise first or CertError("%s: %d association-1 matches seen, stat word 11 (STAT_NMATCH0) says %d" % (
            tag, len(splits[0][0]), int(fr["stat"][11])))

    def _chain(self, fr, pool, unconf, hi, lo, tracked0, a1, a2, up_unc, C1, t1, t3):
        tag, kind, st = self._ctx["tag"], self.kind, self.stats
        if fr["stat"] is not None and len(a1) != int(fr["stat"][11]):
            raise CertError("%s: %d association-1 matches, stat word 11 (STAT_NMATCH0) says %d" % (tag, len(a1), int(fr["stat"][11])))
        pr = {s: k for k, s in enumerate(pool)}
        hc = {d: k for k, d in enumerate(hi.tolist())}
        p1 = [(pr[s], hc[d]) for s, d in a1]
        if kind == "uavmot":
            Ci = self._costs("iou", pool, hi, t1)
            under = Ci[0] < t1
            if under.size:
                under[0, 0] = False
            fused_possible = bool(under.any())             # q20: only a match other than (0, 0) lets the fused solve run
            errs = []
            if fused_possible:
                try:
                    Cf = self._costs("struct", pool, hi, UAV_T1)
                    certify("%s association 1 (fused, 0.8)" % tag, Cf[0], Cf[1], UAV_T1, p1, pool, hi, st.setdefault("assoc1", {}))
                    errs = None
                except CertError as e:
                    errs.append(e)
            if errs is not None:
                if all(p == (0, 0) for p in p1):
                    try:
                        certify("%s association 1 (IoU, 0.7)" % tag, Ci[0], Ci[1], t1, p1, pool, hi, st.setdefault("assoc1", {}))
                        errs = None
                    except CertError as e:
                        errs.append(e)
                if errs is not None:
                    raise errs[0] if errs else CertError("%s: association 1 matched %s, but its IoU solve at 0.7 cannot have matched "
                                                         "a pair other than (0, 0)" % (tag, p1))
        else:
            if C1 is None:
                C1 = self._costs("reid" if self._ctx["feats"] is not None and kind == "botsort" else "iou", pool, hi, t1)
            certify("%s association 1" % tag, C1[0], C1[1], t1, p1, pool, hi, st.setdefault("assoc1", {}))
        m1 = {s for s, _ in a1}
        u1 = set(d for _, d in a1)
        left_hi = np.array([d for d in hi.tolist() if d not in u1], np.int64)
        if kind != "sort":
            if kind in ("bytetrack", "strongsort", "uavmot"):
                r2 = [s for s in pool if s not in m1 and tracked0[s]]
            else:
                r2 = [s for s in pool if s not in m1]
            c2 = left_hi if kind == "strongsort" else lo
            rc = {s: k for k, s in enumerate(r2)}
            cc = {d: k for k, d in enumerate(c2.tolist())}
            for s, d in a2:
                if s not in rc or d not in cc:
                    raise CertError("%s: slot %d updated by detection %d, a pair association 2 does not offer" % (tag, s, d))
            C2 = self._costs("iou", r2, c2, T2)
            certify("%s association 2" % tag, C2[0], C2[1], T2, [(rc[s], cc[d]) for s, d in a2], r2, c2, st.setdefault("assoc2", {}))
            if kind == "strongsort":
                u2 = set(d for _, d in a2)
                left_hi = np.array([d for d in left_hi.tolist() if d not in u2], np.int64)
        elif a2:
            raise CertError("%s: SORT has no association 2, yet %s" % (tag, a2))
        rc = {s: k for k, s in enumerate(unconf)}
        cc = {d: k for k, d in enumerate(left_hi.tolist())}
        for s, d in up_unc:
            if d not in cc:
                raise CertError("%s: unconfirmed slot %d updated by detection %d, which association 3 does not offer" % (tag, s, d))
        how = "dense" if kind == "strongsort" else ("reid" if self._ctx["feats"] is not None and kind == "botsort" else "iou")
        C3 = self._costs(how, unconf, left_hi, t3)
        certify("%s association 3" % tag, C3[0], C3[1], t3, [(rc[s], cc[d]) for s, d in up_unc], unconf, left_hi, st.setdefault("assoc3", {}))

    def _costs(self, how, rows, cols, t):
        cx = self._ctx
        n, m = len(rows), len(cols)
        if n == 0 or m == 0:
            return np.zeros((n, m)), np.zeros((n, m))
        ri = np.array([cx["idx"][s] for s in rows])
        rb = [b.take(ri) for b in cx["rb_all"]]
        cb = cx["colbox"][np.asarray(cols, np.int64)]
        if how == "iou":
            return iou_costs(rb, cb, self.f32)[0]
        if how == "reid":
            tf = np.stack([cx["before"][s]["feat"] for s in rows])
            return reid_costs(rb, cb, tf, cx["feats"][np.asarray(cols, np.int64)], self.f32, self.theta_iou, self.theta_emb)
        if how == "dense":
            tf = np.stack([cx["before"][s]["feat"] for s in rows])
            return strongsort_costs(rb, cb, tf, cx["feats"][np.asarray(cols, np.int64)], self.f32, self.gamma)
        tlwh = K.tlbr_to_tlwh_f32(cx["dets"][np.asarray(cols, np.int64), :4])
        return uavmot_costs(rb, cb, cx["base_mean"], ri, tlwh, cx["tag"])


def report(stats):
    """one line: per association the largest interval width (absolute, relative to U) and the smallest slack of (b)"""
    out = []
    for a in ("assoc1", "assoc2", "assoc3"):
        s = stats.get(a)
        if s:
            out.append("%s: %d solves, %d pairs, width %.3g (rel %.3g), slack %.3g" % (
                a, s.get("assoc", 0), s.get("pairs", 0), s.get("max_width", 0.0), s.get("max_rel_width", 0.0), s.get("min_slack", np.inf)))
    return "; ".join(out)


def spill_bound(f32):
    """association-1 edges that cannot all live in the 227 KB of shared memory the mirror and the second window share"""
    return 227 * 1024 // (8 + (4 if f32 else 8))


# ---------------------------------------------------------------- crowded streams
def crowd_stream(seed, n_frames, n_obj=500, img=700, feat_dim=32, feat_noise=0.3, feat_spread=None, warp_sigma=0.0, miss=0.05):
    """(frames, feats, warps): n_obj objects of 20 - 80 x 40 - 160 px moving inside an img x img area (make_stream's motion; one
    random unit identity feature per object -- with feat_spread, a common unit row plus feat_spread times a random unit row,
    normalised, so that every pair of objects lies close -- and its detections' features that row plus feat_noise times a random
    unit row, normalised), rows sorted by descending score.  Exact duplicate boxes are dropped (the frame check needs exactly one
    detection to explain each update and birth)."""
    rng = np.random.default_rng(seed)
    cx, cy = rng.uniform(100, img - 100, n_obj), rng.uniform(100, img - 100, n_obj)
    w, h = rng.uniform(20, 80, n_obj), rng.uniform(40, 160, n_obj)
    vx, vy = rng.normal(0, 1, n_obj), rng.normal(0, 1, n_obj)
    cls = rng.integers(0, 3, n_obj).astype(np.float32)
    unit = lambda a: a / np.linalg.norm(a, axis=-1, keepdims=True)      # noqa: E731
    ident = unit(rng.normal(0, 1, (n_obj, feat_dim)))
    if feat_spread is not None:
        ident = unit(unit(rng.normal(0, 1, feat_dim)) + feat_spread * ident)
    frames, feats = [], []
    warps = np.zeros((n_frames, 2, 3))
    warps[:, 0, 0] = warps[:, 1, 1] = 1.0
    cam = np.zeros(2)
    for f in range(n_frames):
        cx += vx
        cy += vy
        vx[(cx < 60) | (cx > img - 60)] *= -1
        vy[(cy < 60) | (cy > img - 60)] *= -1
        if warp_sigma > 0:
            t = rng.normal(0, warp_sigma, 2)
            warps[f, :, 2] = t
            cam += t
        jit = rng.normal(0, 1, (n_obj, 4))
        score = rng.uniform(0.05, 0.95, n_obj).astype(np.float32)
        keep = rng.uniform(0, 1, n_obj) >= miss
        box = np.stack([cx - w / 2 + jit[:, 0] + cam[0], cy - h / 2 + jit[:, 1] + cam[1],
                        cx + w / 2 + jit[:, 2] + cam[0], cy + h / 2 + jit[:, 3] + cam[1]], 1)
        box = np.round(np.clip(box, 0, img))
        ok = keep & ((box[:, 2] - box[:, 0]) >= 4) & ((box[:, 3] - box[:, 1]) >= 4)
        _, first = np.unique(box, axis=0, return_index=True)
        uniq = np.zeros(n_obj, bool)
        uniq[first] = True
        ok &= uniq
        fe = unit(ident + feat_noise * unit(rng.normal(0, 1, ident.shape)))
        d = np.concatenate([box[ok], score[ok, None], cls[ok, None]], 1).astype(np.float32)
        order = np.argsort(-d[:, 4], kind="stable")
        frames.append(np.ascontiguousarray(d[order]))
        feats.append(np.ascontiguousarray(fe[ok][order].astype(np.float32)))
    return frames, feats, warps


CROWDS = {
    # kind: (tracker kind, feature dim, crowd_stream keyword arguments)
    "reid": ("botsort", 32, dict(n_obj=760, img=700, feat_noise=0.3, warp_sigma=2.0)),
    "strongsort": ("strongsort", 32, dict(n_obj=260, img=1000, feat_noise=0.1, feat_spread=0.25, warp_sigma=2.0)),
    "uavmot": ("uavmot", 0, dict(n_obj=760, img=700)),
    "bytetrack": ("bytetrack", 0, dict(n_obj=760, img=700)),
    "botsort": ("botsort", 0, dict(n_obj=760, img=700, warp_sigma=2.0)),
}


def crowd_case(name, n_frames, seed=77):
    """(kind, fmt, frames, feats, warps, tracker kwargs) of a crowded stream whose association 1 spills past shared memory"""
    kind, D, kw = CROWDS[name]
    frames, feats, warps = crowd_stream(seed, n_frames, feat_dim=max(D, 4), **kw)
    fmt = {"botsort": "botsort", "strongsort": "strongsort"}.get(kind, "default")
    return (kind, fmt, frames, feats if D else None, warps if kind in ("botsort", "strongsort") else None,
            dict(track_buffer=30, feat_dim=D, cap=1024, dmax=768, ecap=262144))
