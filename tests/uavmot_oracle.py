"""Oracle for UAVMOT (``UAVMOT.update``, tracker/uavmot.py:106-279, appearance off as hard-coded at :76), the CPU statement the fused
kernel's UAVMOT kind (B2T_UAVMOT) and the structure entries (b2t_structure_vectors / b2t_structure_distance) are checked against.

TEST INFRASTRUCTURE.  ``UavmotOracle`` reuses ``oracle.trackers.TrackerOracle``'s track records, Kalman steps and list algebra and
restates the policy line by line:
  * :134-135 high rows score >= det_thresh, low rows low_thresh < score < det_thresh (float32 compares); no camera-motion step;
  * :173-190 association 1, pool x high: IoU distance at 0.7; q20 -- only if that solve's matches array has a non-zero entry (not
    when it is empty or the single pair (0, 0)) is the pool re-solved on 0.98 * IoU distance + (1 - 0.98) * S at 0.8, replacing it;
  * :211-224 association 2, the Tracked leftovers x the low rows, IoU at 0.5; q21 (:228-231) marks strack_pool[idx] lost for every
    unmatched row idx -- an index into u_tracks0;
  * :234-252 association 3, unconfirmed x association 1's leftover high rows at 0.7; births from its leftovers with
    score > det_thresh + 0.1 (float32); then the pruning of the old lost list and the list algebra.
Structure vectors (q22, matching.py:344-386) and S (matching.py:311-320) are restated from the arithmetic, not called:
  * a track point is mean[0:2] in float64 and its neighbour length sqrt(fma(dy, dy, dx * dx)) -- NumPy's 2-element norm goes through
    BLAS ddot, whose tail is one multiply and one fused multiply-add (the fma comes from the C library here);
  * a detection point is get_xy() = tl + wh // 2 in float32 and its length sqrt(dx * dx + dy * dy) in float32 operations;
  * neighbours are the points at 0 < length < 400, the first index wins ties of the maximum and of the minimum;
  * each direction is int(math.atan2(dy, dx) * 180 / math.pi); S is 1 - clip(u.v / (|u| |v|)) in SciPy's order, clamped at 0."""
import ctypes
import ctypes.util
import math

import numpy as np

from oracle.iou import iou_distance_tlbr
from oracle.lapjv import linear_assignment
from oracle.trackers import TrackerOracle, TRACKED, LOST
from oracle import kalman as K

_libm = ctypes.CDLL(ctypes.util.find_library("m"))
_libm.fma.restype = ctypes.c_double
_libm.fma.argtypes = [ctypes.c_double] * 3
LOCAL_R = 400
LAMBDA = 0.98


def _len64(dx, dy):
    return math.sqrt(_libm.fma(dy, dy, dx * dx))


def direction(dx, dy):
    return int(math.atan2(dy, dx) * 180 / math.pi)


def included_angle(v1, v2):
    a1, a2 = direction(float(v1[0]), float(v1[1])), direction(float(v2[0]), float(v2[1]))
    if a1 * a2 >= 0:
        return abs(a1 - a2)
    inc = abs(a1) + abs(a2)
    return 360 - inc if inc > 180 else inc


def lengths(pts, detection):
    """(n, n) neighbour lengths |A - B| in the precision the reference uses for the set"""
    pts = np.asarray(pts, np.float32 if detection else np.float64).reshape(-1, 2)
    dx = pts[:, None, 0] - pts[None, :, 0]
    dy = pts[:, None, 1] - pts[None, :, 1]
    if detection:
        return np.sqrt(dx * dx + dy * dy)
    n = len(pts)
    out = np.empty((n, n))
    for i in range(n):
        for j in range(n):
            out[i, j] = _len64(float(dx[i, j]), float(dy[i, j]))
    return out


def structure_vectors(pts, detection=False, info=None):
    """(n, 3) float64 structure vectors of the points (n, 2).  info (a dict) collects what happened, for the golden's checks: ties of
    the maximum / minimum, lengths at and just inside 400, isolated and single-neighbour points, axis / diagonal directions, and
    the margins (closest non-tied length, closest angle to an integer off the 45-degree multiples)."""
    pts = np.asarray(pts, np.float32 if detection else np.float64).reshape(-1, 2)
    n = len(pts)
    out = np.zeros((n, 3))
    if n == 0:
        return out
    L = lengths(pts, detection)
    for i in range(n):
        row = L[i]
        nb = np.nonzero((row < LOCAL_R) & (row > 0))[0]
        if info is not None:
            info["on400"] = info.get("on400", 0) + int((row == LOCAL_R).sum())
            info["inside400"] = info.get("inside400", 0) + int(((row < LOCAL_R) & (row > LOCAL_R - 2)).sum())
            near = (row != LOCAL_R) & (np.abs(row.astype(np.float64) - LOCAL_R) <= 1e-9 * LOCAL_R)
            info["near400"] = info.get("near400", 0) + int(near.sum())
        if len(nb) == 0:
            out[i] = (1e-4, 1e-4, 1e-4)
            if info is not None:
                info["isolated"] = info.get("isolated", 0) + 1
            continue
        lv = row[nb]
        lmax, lmin = lv.max(), lv.min()
        jmax, jmin = nb[int(np.argmax(lv == lmax))], nb[int(np.argmax(lv == lmin))]
        if info is not None:
            info["tie_max"] = info.get("tie_max", 0) + int((lv == lmax).sum() > 1)
            info["tie_min"] = info.get("tie_min", 0) + int((lv == lmin).sum() > 1)
            for ext in (lmax, lmin):
                other = lv[lv != ext].astype(np.float64)
                if len(other):
                    gap = np.abs(other - float(ext)).min() / float(ext)
                    info["len_gap"] = min(info.get("len_gap", 1.0), gap)
        if lmax == lmin:
            out[i] = (float(lmax), float(lmin), 1e-4)
            if info is not None:
                info["single"] = info.get("single", 0) + int(len(nb) == 1)
            continue
        v1, v2 = pts[jmax] - pts[i], pts[jmin] - pts[i]
        if info is not None:
            for v in (v1, v2):
                dx, dy = float(v[0]), float(v[1])
                if dx == 0 or dy == 0:
                    info["axis"] = info.get("axis", 0) + 1
                elif abs(dx) == abs(dy):
                    info["diag"] = info.get("diag", 0) + 1
                else:
                    a = math.atan2(dy, dx) * 180 / math.pi
                    info["angle_gap"] = min(info.get("angle_gap", 1.0), abs(a - round(a)))
        out[i] = (float(lmax), float(lmin), included_angle(v1, v2))
    return out


def structure_distance(a, b):
    """max(0, cdist(a, b, 'cosine')) in SciPy's order of operations"""
    a = np.asarray(a, np.float64).reshape(-1, 3)
    b = np.asarray(b, np.float64).reshape(-1, 3)
    nu = np.sqrt(a[:, 0] * a[:, 0] + a[:, 1] * a[:, 1] + a[:, 2] * a[:, 2])
    nv = np.sqrt(b[:, 0] * b[:, 0] + b[:, 1] * b[:, 1] + b[:, 2] * b[:, 2])
    s = a[:, None, 0] * b[None, :, 0] + a[:, None, 1] * b[None, :, 1] + a[:, None, 2] * b[None, :, 2]
    c = s / (nu[:, None] * nv[None, :])
    c = np.where(np.abs(c) > 1, np.copysign(1.0, c), c)
    return np.maximum(0.0, 1.0 - c)


def det_centres(tlwh_f32):
    """AMF_STrack.get_xy(): tl + wh // 2 in float32 (q2)"""
    t = np.asarray(tlwh_f32, np.float32).reshape(-1, 4)
    return t[:, :2] + t[:, 2:] // np.float32(2)


class UavmotOracle(TrackerOracle):
    def __init__(self, kalman_format="default", **kw):
        super().__init__(kind="bytetrack", kalman_format=kalman_format, use_gmc=False, **kw)
        self.kind = "uavmot"
        self.events = {}
        self.info = {}
        self.costs = []          # (matrix, threshold) of every assignment of the last frame

    def _la(self, cost, thresh):
        self.costs.append((np.asarray(cost, np.float64), thresh))
        return linear_assignment(cost, thresh)

    def update(self, dets, warp=None):
        trk = self.trk
        self.frame_id += 1
        f = self.frame_id
        self.costs = []
        dets = np.asarray(dets, dtype=np.float32).reshape(-1, 6)
        sc = dets[:, 4]
        tlwh = K.tlbr_to_tlwh_f32(dets[:, :4])
        area = np.isfinite(dets[:, :4]).all(1) & (tlwh[:, 3] != 0)       # as TrackerOracle.update (a deliberate divergence)
        if self.fmt == K.FMT_XYWH:
            area &= tlwh[:, 2] != 0
        him = sc >= np.float32(self.det_thresh)
        lom = ~him & (sc > np.float32(self.low_thresh))
        hi, lo = np.nonzero(him & area)[0], np.nonzero(lom & area)[0]
        tlbr = tlwh.copy()
        tlbr[:, 2:] += tlbr[:, :2]
        tlbr64 = tlbr.astype(np.float64)
        new_thresh = np.float32(self.det_thresh + 0.1)

        unconfirmed = [s for s in self.tracked if not trk[s].activated]
        confirmed = [s for s in self.tracked if trk[s].activated]
        have = {trk[s].tid for s in confirmed}
        pool = confirmed + [s for s in self.lost if trk[s].tid not in have]
        self._predict_pool(pool)

        lost_now, removed_now, births, refind, activated = [], [], [], [], []
        ev = dict(s_decides=0, q20_skip=0, fused=0, q21_updated=0)

        def cols(idx):
            return tlbr64[idx] if len(idx) else np.zeros((0, 4))

        # ---- association 1
        iou1 = iou_distance_tlbr(self._tlbr64(pool), cols(hi))
        m0, ut0, ud0 = self._la(iou1, 0.7)
        m0 = np.asarray(m0)
        if m0.any():
            tp = np.array([np.asarray(trk[s].mean, np.float64)[:2] for s in pool]).reshape(-1, 2)
            S = structure_distance(structure_vectors(tp, False, self.info), structure_vectors(det_centres(tlwh[hi]), True, self.info))
            fused = LAMBDA * iou1 + (1 - LAMBDA) * S
            m0, ut0, ud0 = self._la(fused, 0.8)
            ref, _, _ = linear_assignment(iou1, 0.8 / 0.98)
            ev["fused"] = 1
            ev["s_decides"] = int(sorted(map(tuple, np.asarray(m0).reshape(-1, 2).tolist())) != sorted(map(tuple, np.asarray(ref).reshape(-1, 2).tolist())))
        elif len(m0):
            ev["q20_skip"] = 1
        for it, idt in np.asarray(m0).reshape(-1, 2):
            s, d = pool[it], hi[idt]
            if trk[s].state == TRACKED:
                self._update(s, tlwh[d], sc[d], f)
                activated.append(s)
            elif trk[s].state == LOST:
                self._re_activate(s, tlwh[d], sc[d], f)
                refind.append(s)
        u_tracks0 = [pool[i] for i in ut0 if trk[pool[i]].state == TRACKED]
        u_dets0 = [hi[i] for i in ud0]

        # ---- association 2: Tracked leftovers x low rows; q21
        m1, ut1, _ = self._la(iou_distance_tlbr(self._tlbr64(u_tracks0), cols(lo)), 0.5)
        for it, idt in m1:
            self._update(u_tracks0[it], tlwh[lo[idt]], sc[lo[idt]], f)
            activated.append(u_tracks0[it])
        for idx in ut1:
            s = pool[idx]
            ev["q21_updated"] += int(trk[s].frame_id == f)
            trk[s].state = LOST
            lost_now.append(s)

        # ---- association 3: unconfirmed x association 1's leftovers
        m2, ut2, ud2 = self._la(iou_distance_tlbr(self._tlbr64(unconfirmed), cols(u_dets0)), 0.7)
        for it, idt in m2:
            self._update(unconfirmed[it], tlwh[u_dets0[idt]], sc[u_dets0[idt]], f)
            activated.append(unconfirmed[it])
        for it in ut2:
            self._mark_removed(unconfirmed[it], f, removed_now)
        for i in ud2:
            d = u_dets0[i]
            if sc[d] > new_thresh:
                s = self._birth(tlwh[d], sc[d], dets[d, 5], f)
                births.append(s)
                activated.append(s)

        for s in self.lost:
            if f - trk[s].frame_id > self.max_time_lost:
                self._mark_removed(s, f, removed_now)

        self.events = ev
        self.last_stats = dict(pool=len(pool), hi=len(hi), lo=len(lo), unconfirmed=len(unconfirmed), m0=len(m0), births=len(births))
        return self._emit(self._finish(f, lost_now, removed_now, activated, refind))
