"""Oracle for StrongSORT (``StrongSORT.update``, tracker/strongsort.py:91-250), the CPU statement the fused kernel's StrongSORT kind
(B2T_STRONGSORT) is checked against.

TEST INFRASTRUCTURE.  ``StrongSortOracle`` reuses ``oracle.trackers.TrackerOracle``'s track records, Kalman steps and list algebra
(``_finish`` is joint_stracks / sub_stracks / remove_duplicate_stracks by id) and restates the policy line by line:
  * :118 the detections are the rows with score > det_thresh (float32 compare), each with the raw feature the extractor returned;
  * :140-147 the camera warp (ECC) is applied to the pool only (confirmed ++ lost), BEFORE the prediction;
  * :150-172 association 1, pool x detections: gamma * IoU distance + (1 - gamma) * max(0, cdist(track.features[-1], det feature))
    in float64, thresh 0.7; a Tracked track is updated (Kalman with the score, feature EMA), a Lost one re-activated (no EMA);
  * :176-191 association 2, the Tracked leftovers x the leftover detections, IoU only, thresh 0.5 (updates smooth the feature too);
  * :195-198 q18: ``strack_pool[idx]`` is marked lost for every unmatched row idx of association 2 -- an index into u_tracks0, not
    into the pool;
  * :201-223 association 3, unconfirmed x association 2's leftover detections, fused cost, thresh 0.7; unmatched unconfirmed tracks
    are removed; a leftover with score > det_thresh + 0.1 (float32) is born with its raw feature;
  * :226-240 long-lost pruning over the old lost list, then the list algebra with activated_starcks in its append order.
q19: a track's feature is raw until its first update and unit length after it, so association 1 mostly compares raw detection rows
with unit track rows.  Pinned against the unmodified reference by tests/golden/loop_strongsort.npz
(tests/golden/make_golden_strongsort.py)."""
import numpy as np
from scipy.spatial.distance import cdist

from oracle.iou import iou_distance_tlbr
from oracle.lapjv import linear_assignment
from oracle.trackers import TrackerOracle, TRACKED, LOST
from oracle import kalman as K
from reid_track_oracle import smooth_feature


def euclidean_distance(track_feats, det_feats):
    """matching.embedding_distance(metric='euclidean') (matching.py:92-98) on lists of feature rows."""
    if len(track_feats) == 0 or len(det_feats) == 0:
        return np.zeros((len(track_feats), len(det_feats)), dtype=np.float64)
    a = np.asarray(track_feats, dtype=np.float64)
    b = np.asarray(det_feats, dtype=np.float64)
    return np.maximum(0.0, cdist(a, b))


class StrongSortOracle(TrackerOracle):
    def __init__(self, gamma=0.1, use_ecc=True, kalman_format="strongsort", **kw):
        super().__init__(kind="bytetrack", kalman_format=kalman_format, use_gmc=False, **kw)
        self.kind = "strongsort"
        self.gamma, self.use_ecc = gamma, use_ecc
        self.feat = {}                  # slot -> float32 feature (track.features[-1])
        self.last_active = []
        self.events = {}

    def _fused(self, rows, cols, tlbr64, feats):
        iou = iou_distance_tlbr(self._tlbr64(rows), tlbr64[cols] if len(cols) else np.zeros((0, 4)))
        app = euclidean_distance([self.feat[s] for s in rows], [feats[d] for d in cols])
        return iou, self.gamma * iou + (1. - self.gamma) * app

    def update(self, dets, feats, warp=None):
        """One frame.  feats: (n, D) float32 rows aligned with dets (only the rows with score > det_thresh are read)."""
        trk = self.trk
        self.frame_id += 1
        f = self.frame_id
        dets = np.asarray(dets, dtype=np.float32).reshape(-1, 6)
        feats = np.asarray(feats, dtype=np.float32).reshape(len(dets), -1)
        sc = dets[:, 4]
        tlwh = K.tlbr_to_tlwh_f32(dets[:, :4])
        area = np.isfinite(dets[:, :4]).all(1) & (tlwh[:, 3] != 0)       # as TrackerOracle.update (a deliberate divergence)
        if self.fmt == K.FMT_XYWH:
            area &= tlwh[:, 2] != 0
        hi = np.nonzero((sc > np.float32(self.det_thresh)) & area)[0]
        tlbr = tlwh.copy()
        tlbr[:, 2:] += tlbr[:, :2]
        tlbr64 = tlbr.astype(np.float64)
        new_thresh = np.float32(self.det_thresh + 0.1)

        unconfirmed = [s for s in self.tracked if not trk[s].activated]
        confirmed = [s for s in self.tracked if trk[s].activated]
        have = {trk[s].tid for s in confirmed}
        pool = confirmed + [s for s in self.lost if trk[s].tid not in have]
        if self.use_ecc and warp is not None:
            self._gmc(pool, warp)
        self._predict_pool(pool)

        lost_now, removed_now, births, refind, activated = [], [], [], [], []
        ev = dict(zero_iou1=0, zero_iou_react1=0, q18_updated=0, coast=0, zero_iou3=0)

        def update(s, d):
            self._update(s, tlwh[d], sc[d], f)
            self.feat[s] = smooth_feature(self.feat[s], feats[d])
            activated.append(s)

        # ---- association 1: pool x detections, fused cost
        iou1, cost1 = self._fused(pool, hi, tlbr64, feats)
        m0, ut0, ud0 = linear_assignment(cost1, 0.7)
        for it, idt in m0:
            s, d = pool[it], hi[idt]
            ev["zero_iou1"] += int(iou1[it, idt] == 1.0)
            if trk[s].state == TRACKED:
                update(s, d)
            elif trk[s].state == LOST:
                ev["zero_iou_react1"] += int(iou1[it, idt] == 1.0)
                self._re_activate(s, tlwh[d], sc[d], f)
                refind.append(s)

        # ---- association 2: Tracked leftovers x leftover detections, IoU only
        u_tracks0 = [pool[i] for i in ut0 if trk[pool[i]].state == TRACKED]
        u_dets0 = [hi[i] for i in ud0]
        m1, ut1, ud1 = linear_assignment(iou_distance_tlbr(self._tlbr64(u_tracks0), tlbr64[u_dets0] if u_dets0 else np.zeros((0, 4))), 0.5)
        u_det1 = [u_dets0[i] for i in ud1]
        for it, idt in m1:
            update(u_tracks0[it], u_dets0[idt])
        # q18: the index is into u_tracks0, the track marked is the pool's
        for idx in ut1:
            s = pool[idx]
            if trk[s].frame_id == f:
                ev["q18_updated"] += 1
            trk[s].state = LOST
            lost_now.append(s)
        ev["coast"] = sum(1 for i in ut1 if trk[u_tracks0[i]].state == TRACKED)

        # ---- association 3: unconfirmed x association 2's leftovers, fused cost
        iou3, cost3 = self._fused(unconfirmed, u_det1, tlbr64, feats)
        m2, ut2, ud2 = linear_assignment(cost3, 0.7)
        for it, idt in m2:
            ev["zero_iou3"] += int(iou3[it, idt] == 1.0)
            update(unconfirmed[it], u_det1[idt])
        for it in ut2:
            self._mark_removed(unconfirmed[it], f, removed_now)
        for i in ud2:
            d = u_det1[i]
            if sc[d] > new_thresh:
                s = self._birth(tlwh[d], sc[d], dets[d, 5], f)
                self.feat[s] = feats[d].copy()
                births.append(s)
                activated.append(s)

        # ---- long-lost pruning (the old lost list)
        for s in self.lost:
            if f - trk[s].frame_id > self.max_time_lost:
                self._mark_removed(s, f, removed_now)

        self.events = ev
        self.last_stats = dict(pool=len(pool), hi=len(hi), unconfirmed=len(unconfirmed), m0=len(m0), births=len(births))
        active = self._finish(f, lost_now, removed_now, activated, refind)
        for s in list(self.feat):
            if s not in trk:
                del self.feat[s]
        self.last_active = active
        return self._emit(active)

    def update_without_detection(self):
        res = super().update_without_detection()
        self.last_active = [s for s in self.tracked if self.trk[s].activated]
        return res

    def last_features(self):
        """(n, D) float32: the features of the tracks the last update returned, in its row order."""
        return np.array([self.feat[s] for s in self.last_active], dtype=np.float32)
