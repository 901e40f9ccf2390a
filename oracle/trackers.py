"""Oracle: per-frame association state machines of the reference (SORT / ByteTrack / BoT-SORT).

TEST INFRASTRUCTURE (see oracle/__init__.py).  Restates, on slot-indexed arrays and index
lists (the layout the CUDA kernel uses), the behaviour of
  * ``BaseTracker.update``           tracker/basetrack.py:368-487   (kind='sort')
  * ``ByteTrack.update``             tracker/bytetrack.py:41-204    (kind='bytetrack')
  * ``BoTSORT.update`` + ``multi_gmc`` tracker/botsort.py:313-493, :250-269 (kind='botsort')
  * ``STrack`` life cycle            tracker/basetrack.py:222-339
  * ``joint_stracks / sub_stracks / remove_duplicate_stracks``  tracker/basetrack.py:540-576
including the quirks SURVEY.md section 8a lists (q2-q8, q13).  Pinned against the reference
classes themselves run through oracle/refshim.py (tests/golden/loop_*.npz).

Appearance (ReID) branches are off, as in the reference defaults (bytetrack.py:11).
"""
import numpy as np

from . import kalman as K
from .iou import iou_distance_tlbr
from .lapjv import linear_assignment

NEW, TRACKED, LOST, REMOVED = 0, 1, 2, 3


class IdCounter:
    """BaseTrack._count (basetrack.py:22,43-46): process-global, shared by every tracker (q8)."""

    def __init__(self, start=0):
        self.count = start

    def next_id(self):
        self.count += 1
        return self.count


class _Trk:
    __slots__ = ("tid", "state", "activated", "tracklet_len", "start_frame", "frame_id", "cls", "score",
                 "mean", "cov", "mean_f32", "removed_at")


class TrackerOracle:
    def __init__(self, kind="bytetrack", conf_thresh=0.2, track_buffer=30, frame_rate=30,
                 kalman_format=None, iou_thresh=0.5, use_gmc=True, ids=None):
        assert kind in ("sort", "bytetrack", "botsort")
        self.kind = kind
        if kalman_format is None:
            kalman_format = "botsort" if kind == "botsort" else "default"  # track.py:68-69
        self.fmt = K.FMT_BY_NAME[kalman_format]
        self.det_thresh = conf_thresh                                   # basetrack.py:354
        self.low_thresh = max(0.15, conf_thresh - 0.3)                  # bytetrack.py:15
        self.iou_thresh = iou_thresh
        self.max_time_lost = int(frame_rate / 30.0 * track_buffer)     # basetrack.py:355-356
        self.use_gmc = use_gmc and kind == "botsort"
        self.ids = ids if ids is not None else IdCounter()
        self.frame_id = 0
        self.trk = {}          # slot -> _Trk   (slot numbers are never reused in the oracle)
        self._next_slot = 0
        self.tracked = []      # self.tracked_stracks (order matters, q13)
        self.lost = []         # self.lost_stracks
        self.removed_ids = set()   # ids ever appended to self.removed_stracks
        self.removed_now_ids = []  # ids appended to self.removed_stracks by the last frame, in order (a track can recur)
        self.last_stats = {}

    # ------------------------------------------------------------------ helpers
    def _tlwh(self, s):
        t = self.trk[s]
        return K.mean_to_tlwh(self.fmt, t.mean[:4].astype(np.float32) if t.mean_f32 else t.mean[:4])

    def _tlbr64(self, slots):
        out = np.zeros((len(slots), 4), dtype=np.float64)
        for k, s in enumerate(slots):
            r = self._tlwh(s)
            r[2:] += r[:2]
            out[k] = r
        return out

    def _kf_update(self, s, det_tlwh_f32, score):
        t = self.trk[s]
        z = K.tlwh_to_meas_f32(self.fmt, det_tlwh_f32)
        conf = score if self.fmt == K.FMT_NSA else 0.0
        t.mean, t.cov = K.update(self.fmt, t.mean, t.cov, z, mean_f32=t.mean_f32, confidence=conf)
        t.mean_f32 = False

    def _update(self, s, det_tlwh_f32, score, f):          # STrack.update, basetrack.py:296-339
        t = self.trk[s]
        t.frame_id = f
        t.tracklet_len += 1
        t.score = score
        self._kf_update(s, det_tlwh_f32, score)
        t.state, t.activated = TRACKED, True

    def _re_activate(self, s, det_tlwh_f32, score, f):     # STrack.re_activate, basetrack.py:273-294 (q7)
        t = self.trk[s]
        z = K.tlwh_to_meas_f32(self.fmt, det_tlwh_f32)
        t.mean, t.cov = K.update(self.fmt, t.mean, t.cov, z, mean_f32=t.mean_f32, confidence=0.0)
        t.mean_f32 = False
        t.tracklet_len = 0
        t.state, t.activated = TRACKED, True
        t.frame_id = f
        t.score = score

    def _birth(self, det_tlwh_f32, score, cls, f):         # STrack.activate, basetrack.py:222-245 (q5)
        t = _Trk()
        t.tid = self.ids.next_id()
        z = K.tlwh_to_meas_f32(self.fmt, det_tlwh_f32)
        t.mean, t.cov = K.initiate(self.fmt, z)
        t.mean_f32 = True
        t.state = TRACKED
        t.activated = (f == 1)
        t.frame_id = t.start_frame = f
        t.tracklet_len = 0
        t.cls, t.score = cls, score
        t.removed_at = None
        s = self._next_slot
        self._next_slot += 1
        self.trk[s] = t
        return s

    def _predict_pool(self, pool):                         # STrack.multi_predict, basetrack.py:253-271 (q6)
        if not pool:
            return
        all_f32 = all(self.trk[s].mean_f32 for s in pool)
        means = np.stack([self.trk[s].mean.astype(np.float32 if all_f32 else np.float64) for s in pool])
        covs = np.stack([np.asarray(self.trk[s].cov, dtype=np.float64) for s in pool])
        for k, s in enumerate(pool):
            if self.trk[s].state != TRACKED:
                means[k, 7] = 0
        means, covs = K.multi_predict(self.fmt, means, covs, all_f32=all_f32)
        for k, s in enumerate(pool):
            t = self.trk[s]
            t.mean, t.cov, t.mean_f32 = means[k], covs[k], False

    def _gmc(self, slots, warp):                           # multi_gmc, botsort.py:250-269
        if not slots:
            return
        means = np.stack([np.asarray(self.trk[s].mean, dtype=np.float64) for s in slots])
        covs = np.stack([np.asarray(self.trk[s].cov, dtype=np.float64) for s in slots])
        means, covs = K.gmc_apply(means, covs, warp)
        for k, s in enumerate(slots):
            t = self.trk[s]
            t.mean, t.cov, t.mean_f32 = means[k], covs[k], False

    def _mark_removed(self, s, f, removed_now):
        self.trk[s].state = REMOVED
        removed_now.append(s)

    # ------------------------------------------------------------------ list algebra
    def _finish(self, f, lost_now, removed_now, births, refind):
        trk = self.trk
        self.removed_now_ids = [trk[s].tid for s in removed_now]
        tracked = [s for s in self.tracked if trk[s].state == TRACKED]
        have = {trk[s].tid for s in tracked}
        for s in births + refind:                           # joint_stracks x2 (activated ones already present)
            if trk[s].tid not in have:
                have.add(trk[s].tid)
                tracked.append(s)
        # sub_stracks(lost, tracked): dict keyed by id keeps first position
        lost, seen = [], set()
        for s in self.lost:
            tid = trk[s].tid
            if tid in seen:
                continue
            seen.add(tid)
            if tid not in have:
                lost.append(s)
        lost = lost + lost_now
        # sub_stracks(lost, self.removed_stracks) -- removed list as of the END of the previous frame
        out, seen = [], set()
        for s in lost:
            tid = trk[s].tid
            if tid in seen:
                continue
            seen.add(tid)
            if tid not in self.removed_ids:
                out.append(s)
        lost = out
        for s in removed_now:
            self.removed_ids.add(trk[s].tid)
        # remove_duplicate_stracks (basetrack.py:563-576)
        if tracked and lost:
            pd = iou_distance_tlbr(self._tlbr64(tracked), self._tlbr64(lost))
            dupa, dupb = set(), set()
            for p, q in zip(*np.where(pd < 0.15)):
                tp = trk[tracked[p]].frame_id - trk[tracked[p]].start_frame
                tq = trk[lost[q]].frame_id - trk[lost[q]].start_frame
                if tp > tq:
                    dupb.add(q)
                else:
                    dupa.add(p)
            tracked = [s for i, s in enumerate(tracked) if i not in dupa]
            lost = [s for i, s in enumerate(lost) if i not in dupb]
        self.tracked, self.lost = tracked, lost
        live = set(tracked) | set(lost)
        for s in list(trk):
            if s not in live:
                del trk[s]
        return [s for s in tracked if trk[s].activated]

    def list_rows(self, which):
        """``tracked_stracks`` / ``lost_stracks`` in list order: (int rows id, state, is_activated, start_frame, frame_id,
        tracklet_len; float64 tlwh)."""
        slots = self.tracked if which == "tracked" else self.lost
        rows = np.array([[self.trk[s].tid, self.trk[s].state, int(self.trk[s].activated), self.trk[s].start_frame,
                          self.trk[s].frame_id, self.trk[s].tracklet_len] for s in slots], np.int64).reshape(-1, 6)
        tlwh = np.array([np.asarray(self._tlwh(s), np.float64) for s in slots]).reshape(-1, 4)
        return rows, tlwh

    def _emit(self, slots):
        out = []
        for s in slots:
            t = self.trk[s]
            out.append((t.tid, np.asarray(self._tlwh(s), dtype=np.float64), float(t.cls), float(t.score)))
        return out

    # ------------------------------------------------------------------ one frame
    def update(self, dets, warp=None):
        trk = self.trk
        self.frame_id += 1
        f = self.frame_id
        dets = np.asarray(dets, dtype=np.float32).reshape(-1, 6)
        sc = dets[:, 4]
        f32 = np.float32
        tlwh = K.tlbr_to_tlwh_f32(dets[:, :4])
        # deliberate divergence, limited to boxes the reference cannot track (as in the kernel): a non-finite coordinate, zero height
        # (xyah: no aspect ratio, zero Kalman noise -> NaN state / failed Cholesky) or, with the xywh filter, zero width takes no part
        area = np.isfinite(dets[:, :4]).all(1) & (tlwh[:, 3] != 0)
        if self.fmt == K.FMT_XYWH:
            area &= tlwh[:, 2] != 0
        if self.kind == "sort":
            hi = np.nonzero(np.logical_and(sc > f32(self.det_thresh), area))[0]  # basetrack.py:387
            lo = np.zeros(0, dtype=np.int64)
        else:
            him = sc >= f32(self.det_thresh)                                    # bytetrack.py:69-70
            lom = np.logical_and(~him, sc > f32(self.low_thresh))
            hi, lo = np.nonzero(np.logical_and(him, area))[0], np.nonzero(np.logical_and(lom, area))[0]
        tlbr = tlwh.copy()
        tlbr[:, 2:] += tlbr[:, :2]
        tlbr64 = tlbr.astype(np.float64)
        new_thresh = f32(self.det_thresh + 0.1)                                 # bytetrack.py:175 in float32

        unconfirmed = [s for s in self.tracked if not trk[s].activated]
        confirmed = [s for s in self.tracked if trk[s].activated]
        have = {trk[s].tid for s in confirmed}
        pool = confirmed + [s for s in self.lost if trk[s].tid not in have]      # joint_stracks
        self._predict_pool(pool)
        if self.use_gmc and warp is not None:
            self._gmc(pool, warp)
            self._gmc(unconfirmed, warp)

        lost_now, removed_now, births, refind = [], [], [], []

        def apply(slot, d):
            st = trk[slot].state
            if st == TRACKED:
                self._update(slot, tlwh[d], sc[d], f)
            elif st == LOST or self.kind == "sort":                              # basetrack.py:424-426 has a bare else
                self._re_activate(slot, tlwh[d], sc[d], f)
                refind.append(slot)

        # ---- association 1: pool x high dets
        t1 = self.iou_thresh if self.kind == "sort" else 0.9
        cost = iou_distance_tlbr(self._tlbr64(pool), tlbr64[hi])
        m0, ut0, ud0 = linear_assignment(cost, t1)
        for it, idt in m0:
            apply(pool[it], hi[idt])
        u_dets0 = [hi[i] for i in ud0]

        if self.kind == "sort":
            for it in ut0:                                                       # basetrack.py:429-433
                if trk[pool[it]].state == TRACKED:
                    trk[pool[it]].state = LOST
                    lost_now.append(pool[it])
        else:
            # ---- association 2: remaining tracks x low dets
            if self.kind == "bytetrack":
                ut = [pool[i] for i in ut0 if trk[pool[i]].state == TRACKED]    # bytetrack.py:131
            else:
                ut = [pool[i] for i in ut0]                                      # botsort.py:411 (q4)
            cost = iou_distance_tlbr(self._tlbr64(ut), tlbr64[lo])
            m1, ut1, _ = linear_assignment(cost, 0.5)
            for it, idt in m1:
                apply(ut[it], lo[idt])
            for it in ut1:                                                       # mark_lost (also re-marks lost ones in botsort)
                trk[ut[it]].state = LOST
                lost_now.append(ut[it])

        # ---- association 3: unconfirmed x leftover high dets
        t3 = self.iou_thresh + 0.1 if self.kind == "sort" else 0.7
        cost = iou_distance_tlbr(self._tlbr64(unconfirmed), tlbr64[u_dets0] if len(u_dets0) else np.zeros((0, 4)))
        m2, ut2, ud2 = linear_assignment(cost, t3)
        for it, idt in m2:
            self._update(unconfirmed[it], tlwh[u_dets0[idt]], sc[u_dets0[idt]], f)
        for it in ut2:
            self._mark_removed(unconfirmed[it], f, removed_now)

        # ---- births (q3: BoT-SORT iterates the first-stage leftovers, bytetrack the third-stage ones)
        birth_dets = u_dets0 if self.kind == "botsort" else [u_dets0[i] for i in ud2]
        for d in birth_dets:
            if sc[d] > new_thresh:
                births.append(self._birth(tlwh[d], sc[d], dets[d, 5], f))

        # ---- step 5: prune long-lost (iterates the OLD lost list)
        for s in self.lost:
            if f - trk[s].frame_id > self.max_time_lost:
                self._mark_removed(s, f, removed_now)

        self.last_stats = dict(pool=len(pool), hi=len(hi), lo=len(lo), unconfirmed=len(unconfirmed),
                               m0=len(m0), births=len(births), refind=len(refind), lost_now=len(lost_now),
                               removed_now=len(removed_now))
        active = self._finish(f, lost_now, removed_now, births, refind)
        return self._emit(active)

    def update_without_detection(self):
        """BaseTracker.update_without_detection, basetrack.py:489-537."""
        trk = self.trk
        self.frame_id += 1
        confirmed = [s for s in self.tracked if trk[s].activated]
        have = {trk[s].tid for s in confirmed}
        pool = confirmed + [s for s in self.lost if trk[s].tid not in have]
        self._predict_pool(pool)
        active = self._finish(self.frame_id, [], [], [], [])
        return self._emit(active)
