"""Oracle for BoT-SORT with appearance features (``use_apperance_model = True``), the CPU statement the fused kernel's
feature path is checked against.

TEST INFRASTRUCTURE.  ``ReidBotsortOracle`` extends ``oracle.trackers.TrackerOracle('botsort')`` by the three places the
reference's ``BoTSORT.update`` uses appearance (tracker/botsort.py:345-349, :386-392, :440-446) and by ``STrack.update``'s feature
EMA (basetrack.py:323-332), with the reference's own NumPy expressions:
  1. the rows with score >= det_thresh (float32 compare) carry the float32 feature the extractor returned, unchanged;
  2. associations 1 and 3: App = 0.5 * (1 - cos) from float64 rows normalised in float64 (matching.py:84-103, 165-178),
     App[IoU_d > theta_iou] = 1, App[App > theta_emb] = 1, cost = min(IoU_d, App); association 2 and the duplicate pass stay IoU;
  3. an update by a high detection smooths the feature in float32; re-activation and low-detection updates leave it; a birth
     stores the raw detection feature (births come from every first-stage leftover, q3).
Pinned against the unmodified reference by tests/golden/loop_botsort_reid.npz (tests/golden/make_golden_reid_track.py)."""
import numpy as np

from oracle.iou import iou_distance_tlbr
from oracle.lapjv import linear_assignment
from oracle.trackers import TrackerOracle, TRACKED, LOST
from oracle import kalman as K


def embedding_distance(track_feats, det_feats):
    """matching.embedding_distance(metric='cosine') with cal_cosine_distance, on lists of feature rows."""
    cost = np.zeros((len(track_feats), len(det_feats)), dtype=np.float64)
    if cost.size == 0:
        return cost
    a = np.asarray(track_feats, dtype=np.float64)
    b = np.asarray(det_feats, dtype=np.float64)
    a = a / np.linalg.norm(a, axis=1, keepdims=True)
    b = b / np.linalg.norm(b, axis=1, keepdims=True)
    return 1. - np.dot(a, b.T)


def smooth_feature(old, det_feat):
    """STrack.update's EMA (basetrack.py:325-329), float32 under NumPy 2."""
    feature = det_feat / np.linalg.norm(det_feat)
    smooth_feat = 0.9 * old + (1 - 0.9) * feature
    smooth_feat /= np.linalg.norm(smooth_feat)
    return smooth_feat


class ReidBotsortOracle(TrackerOracle):
    def __init__(self, theta_iou=0.5, theta_emb=0.25, **kw):
        super().__init__(kind="botsort", **kw)
        self.theta_iou, self.theta_emb = theta_iou, theta_emb      # botsort.py:289
        self.feat = {}                                              # slot -> float32 feature (track.features[-1])
        self.last_costs = []                                        # (IoU_d, App) of associations 1 and 3 of the last frame

    def _fused(self, rows, dets_idx, tlbr64, feats):
        iou = iou_distance_tlbr(self._tlbr64(rows), tlbr64[dets_idx] if len(dets_idx) else np.zeros((0, 4)))
        if feats is None:
            return iou
        app = 0.5 * embedding_distance([self.feat[s] for s in rows], [feats[d] for d in dets_idx])
        self.last_costs.append((iou.copy(), app.copy()))
        app[iou > self.theta_iou] = 1
        app[app > self.theta_emb] = 1
        return np.minimum(iou, app)

    def update(self, dets, warp=None, feats=None):
        """One frame.  feats: (n, D) float32 rows aligned with dets (only the high-score rows are read), or None for the IoU-only
        tracker."""
        trk = self.trk
        self.frame_id += 1
        f = self.frame_id
        self.last_costs = []
        dets = np.asarray(dets, dtype=np.float32).reshape(-1, 6)
        if feats is not None:
            feats = np.asarray(feats, dtype=np.float32)
        sc = dets[:, 4]
        f32 = np.float32
        tlwh = K.tlbr_to_tlwh_f32(dets[:, :4])
        area = np.isfinite(dets[:, :4]).all(1) & (tlwh[:, 3] != 0)
        if self.fmt == K.FMT_XYWH:
            area &= tlwh[:, 2] != 0
        him = sc >= f32(self.det_thresh)
        lom = np.logical_and(~him, sc > f32(self.low_thresh))
        hi, lo = np.nonzero(np.logical_and(him, area))[0], np.nonzero(np.logical_and(lom, area))[0]
        tlbr = tlwh.copy()
        tlbr[:, 2:] += tlbr[:, :2]
        tlbr64 = tlbr.astype(np.float64)
        new_thresh = f32(self.det_thresh + 0.1)

        unconfirmed = [s for s in self.tracked if not trk[s].activated]
        confirmed = [s for s in self.tracked if trk[s].activated]
        have = {trk[s].tid for s in confirmed}
        pool = confirmed + [s for s in self.lost if trk[s].tid not in have]
        self._predict_pool(pool)
        if self.use_gmc and warp is not None:
            self._gmc(pool, warp)
            self._gmc(unconfirmed, warp)

        lost_now, removed_now, births, refind = [], [], [], []

        def update_high(slot, d):
            self._update(slot, tlwh[d], sc[d], f)
            if feats is not None:
                self.feat[slot] = smooth_feature(self.feat[slot], feats[d])

        # ---- association 1: pool x high dets (IoU fused with appearance)
        m0, ut0, ud0 = linear_assignment(self._fused(pool, hi, tlbr64, feats), 0.9)
        for it, idt in m0:
            s, d = pool[it], hi[idt]
            if trk[s].state == TRACKED:
                update_high(s, d)
            elif trk[s].state == LOST:
                self._re_activate(s, tlwh[d], sc[d], f)
                refind.append(s)
        u_dets0 = [hi[i] for i in ud0]

        # ---- association 2: every leftover pool track x low dets, IoU only (q4)
        ut = [pool[i] for i in ut0]
        m1, ut1, _ = linear_assignment(iou_distance_tlbr(self._tlbr64(ut), tlbr64[lo]), 0.5)
        for it, idt in m1:
            s, d = ut[it], lo[idt]
            if trk[s].state == TRACKED:
                self._update(s, tlwh[d], sc[d], f)
            elif trk[s].state == LOST:
                self._re_activate(s, tlwh[d], sc[d], f)
                refind.append(s)
        for it in ut1:
            trk[ut[it]].state = LOST
            lost_now.append(ut[it])

        # ---- association 3: unconfirmed x leftover high dets (fused)
        m2, ut2, _ = linear_assignment(self._fused(unconfirmed, u_dets0, tlbr64, feats), 0.7)
        for it, idt in m2:
            update_high(unconfirmed[it], u_dets0[idt])
        for it in ut2:
            self._mark_removed(unconfirmed[it], f, removed_now)

        # ---- births from every first-stage leftover (q3), with the raw detection feature
        for d in u_dets0:
            if sc[d] > new_thresh:
                s = self._birth(tlwh[d], sc[d], dets[d, 5], f)
                births.append(s)
                if feats is not None:
                    self.feat[s] = feats[d].copy()

        for s in self.lost:
            if f - trk[s].frame_id > self.max_time_lost:
                self._mark_removed(s, f, removed_now)

        self.last_stats = dict(pool=len(pool), hi=len(hi), lo=len(lo), unconfirmed=len(unconfirmed), m0=len(m0), births=len(births))
        active = self._finish(f, lost_now, removed_now, births, refind)
        for s in list(self.feat):
            if s not in trk:
                del self.feat[s]
        self.last_active = active
        return self._emit(active)

    def last_features(self):
        """(n, D) float32: the smoothed features of the tracks the last update returned, in its row order."""
        return np.array([self.feat[s] for s in self.last_active], dtype=np.float32)
