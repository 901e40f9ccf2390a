"""Drop-in for the reference's ``tracker/basetrack.py``: TrackState, BaseTrack, STrack, BaseTracker
(SORT) and the list helpers -- same names, same attributes.

Two ways in:
  * ``BaseTracker.update`` (and ByteTrack / BoTSORT in their modules) runs the whole frame in ONE
    kernel on device-resident state (b200track.engine.TrackEngine, csrc/b2t_step.cuh) and hands back
    ``STrack`` views (``track_id``, ``tlwh``, ``cls``, ``score`` filled; ``mean`` / ``cov`` fetched
    from the device on first access).  ``tracker/track.py:151-164`` only reads tlwh / track_id / cls.
  * ``STrack`` is also a complete stand-alone object (activate / predict / update / re_activate /
    multi_predict with NumPy state) for third-party trackers that drive tracks one by one; its
    arithmetic goes through the GPU Kalman ops in ``kalman_filter``.
"""
from collections import OrderedDict

import numpy as np

import _b2t_path  # noqa: F401
import matching
from kalman_filter import KalmanFilter, NaiveKalmanFilter, BoTSORTKalmanFilter, NSAKalmanFilter
from b200track import _lib as L

import torch  # noqa: E402


class TrackState(object):
    New = 0
    Tracked = 1
    Lost = 2
    Removed = 3


class BaseTrack(object):
    _count = 0                      # process-global id counter, never reset between sequences (q8)

    track_id = 0
    is_activated = False
    state = TrackState.New
    history = OrderedDict()
    features = []
    curr_feature = None
    score = 0
    start_frame = 0
    frame_id = 0
    time_since_update = 0
    location = (np.inf, np.inf)

    @property
    def end_frame(self):
        return self.frame_id

    @staticmethod
    def next_id():
        BaseTrack._count += 1
        return BaseTrack._count

    def activate(self, *args):
        raise NotImplementedError

    def predict(self):
        raise NotImplementedError

    def update(self, *args, **kwargs):
        raise NotImplementedError

    def mark_lost(self):
        self.state = TrackState.Lost

    def mark_removed(self):
        self.state = TrackState.Removed


KALMAN_DICT = {
    'default': KalmanFilter,
    'naive': NaiveKalmanFilter,
    'botsort': BoTSORTKalmanFilter,
    'strongsort': NSAKalmanFilter,
}


class STrack(BaseTrack):
    def __init__(self, cls, tlwh, score, kalman_format='default', feature=None, use_avg_of_feature=True,
                 store_features_budget=100):
        super().__init__()
        self.cls = cls
        self._tlwh = np.asarray(tlwh, dtype=np.float32)
        self.score = score
        self.is_activated = False
        self.tracklet_len = 0
        self.track_id = None
        self.start_frame = None
        self.frame_id = None
        self.time_since_update = None
        self.features = []
        self.store_features_budget = store_features_budget
        self.has_feature = feature is not None
        self.use_avg_of_feature = use_avg_of_feature
        if feature is not None:
            self.features.append(feature)
        self.kalman_format = kalman_format
        self.kalman = KALMAN_DICT[kalman_format]()
        self.mean, self.cov = None, None

    # ---- conversions (same arithmetic, incl. the floor division of tlwh2xywh: q2)
    @staticmethod
    def tlbr2tlwh(tlbr):
        r = np.asarray(tlbr).copy()
        r[2:] -= r[:2]
        return r

    @staticmethod
    def tlwh2xyah(tlwh):
        r = np.asarray(tlwh).copy()
        r[:2] += r[2:] / 2
        r[2] /= r[3]
        return r

    @staticmethod
    def tlwh2xyar(tlwh):
        r = np.asarray(tlwh).copy()
        r[:2] += r[2:] / 2
        r[2] *= r[3]
        r[3] = tlwh[-1] / tlwh[-2]
        return r

    @staticmethod
    def tlwh2xywh(tlwh):
        r = np.asarray(tlwh).copy()
        r[:2] += r[2:] // 2
        return r

    @staticmethod
    def xywh2tlbr(xywh):
        r = np.asarray(xywh).copy()
        r[..., :2] -= r[..., 2:] // 2
        r[..., 2:] = r[..., :2] + r[..., 2:]
        return np.maximum(0.0, r)

    @staticmethod
    def xywh2tlwh(xywh):
        r = np.asarray(xywh).copy()
        r[..., :2] -= r[..., 2:] // 2
        return r

    def _measure(self, tlwh):
        if self.kalman_format in ('default', 'strongsort'):
            return self.tlwh2xyah(tlwh)
        if self.kalman_format == 'naive':
            return self.tlwh2xyar(tlwh)
        if self.kalman_format == 'botsort':
            return self.tlwh2xywh(tlwh)
        raise NotImplementedError

    @property
    def tlwh(self):
        if self.mean is None:
            return self._tlwh.copy()
        r = self.mean[:4].copy()
        if self.kalman_format in ('default', 'strongsort'):
            r[2] *= r[3]
            r[:2] -= r[2:] / 2
        elif self.kalman_format == 'naive':
            r[-1] = np.sqrt(r[-1] * r[-2])
            r[-2] /= r[-1]
        elif self.kalman_format == 'botsort':
            r[:2] -= r[2:] / 2
        else:
            raise NotImplementedError
        return r

    @property
    def tlbr(self):
        r = self.tlwh.copy()
        r[2:] += r[:2]
        return r

    def activate(self, frame_id):
        self.track_id = BaseTrack.next_id()
        self.mean, self.cov = self.kalman.initiate(self._measure(self._tlwh))
        self.state = TrackState.Tracked
        if frame_id == 1:
            self.is_activated = True                    # later births stay unconfirmed for a frame (q5)
        self.frame_id = frame_id
        self.start_frame = frame_id
        self.time_since_update = 0

    def predict(self):
        self.mean, self.cov = self.kalman.predict(self.mean, self.cov)

    @staticmethod
    def multi_predict(stracks, kalman):
        if len(stracks) > 0:
            means = np.asarray([st.mean.copy() for st in stracks])
            covs = np.asarray([st.cov for st in stracks])
            for i, st in enumerate(stracks):
                if st.state != TrackState.Tracked:
                    means[i][-1] = 0                     # q6
            means, covs = kalman.multi_predict(means, covs)
            for st, m, c in zip(stracks, means, covs):
                st.mean, st.cov = m, c
        for st in stracks:
            st.time_since_update += 1

    def re_activate(self, new_track, frame_id, new_id=False):
        self.mean, self.cov = self.kalman.update(self.mean, self.cov, self._measure(new_track.tlwh))
        self.tracklet_len = 0
        self.state = TrackState.Tracked
        self.is_activated = True
        self.frame_id = frame_id
        if new_id:
            self.track_id = self.next_id()
        self.score = new_track.score
        self.time_since_update = 0

    def update(self, new_track, frame_id):
        self.frame_id = frame_id
        self.tracklet_len += 1
        self.score = new_track.score
        z = self._measure(new_track.tlwh)
        if self.kalman_format == 'strongsort':
            self.mean, self.cov = self.kalman.update(self.mean, self.cov, z, self.score)
        else:
            self.mean, self.cov = self.kalman.update(self.mean, self.cov, z)
        if new_track.has_feature:
            feat = new_track.features[0] / np.linalg.norm(new_track.features[0])
            if self.use_avg_of_feature:
                smooth = 0.9 * self.features[-1] + 0.1 * feat
                self.features = [smooth / np.linalg.norm(smooth)]
            else:
                self.features.append(feat)
                self.features = self.features[-self.store_features_budget:]
        self.state = TrackState.Tracked
        self.is_activated = True
        self.time_since_update = 0


class _TrackView(STrack):
    """An ``STrack`` whose numbers come from one row of the fused kernel's state (b2t_tracker_step output rows, or
    b2t_tracker_read_list rows for the lost list).  ``mean`` / ``cov`` are fetched from the device on first access and only while the
    engine is still at the frame this view was created for (afterwards the slot may hold a newer state or another track)."""

    def __init__(self, engine, seq, row, kalman_format, frame_id, state=TrackState.Tracked, extra=None):
        BaseTrack.__init__(self)
        self._engine, self._seq, self._slot = engine, seq, int(row[7])
        self._row = row
        self._view_frame = frame_id
        self.track_id = int(row[0])
        self.cls = np.float32(row[5])
        self.score = np.float32(row[6])
        self.is_activated = True
        self.state = state
        self.frame_id = frame_id
        self.start_frame = frame_id
        self.tracklet_len = 0
        self.time_since_update = 0
        if extra is not None:                                  # state, is_activated, tracklet_len, start_frame, frame_id of the slot
            self.state = int(extra[0])
            self.is_activated = bool(extra[1])
            self.tracklet_len, self.start_frame, self.frame_id = int(extra[2]), int(extra[3]), int(extra[4])
            self.time_since_update = frame_id - self.frame_id
        self.kalman_format = kalman_format
        self._features = None
        self.has_feature = engine.feat_dim > 0
        self._mean = self._cov = None

    @property
    def tlwh(self):
        return self._row[1:5].copy()

    @property
    def _tlwh(self):
        return self._row[1:5].astype(np.float32)

    def _check_frame(self, what):
        if self._engine.np_stat[self._seq, L.STAT_FRAME] != self._view_frame:
            raise RuntimeError("track %d: %s were not read at frame %d and the tracker has moved on (frame %d): read them "
                               "in the frame the track was returned" % (self.track_id, what, self._view_frame, int(self._engine.np_stat[self._seq, L.STAT_FRAME])))

    def _fetch(self):
        if self._mean is None:
            self._check_frame("mean / cov")
            self._mean, self._cov = self._engine.read_slot(self._seq, self._slot)

    @property
    def features(self):
        """[smoothed appearance feature] (BoT-SORT with ReID, read from the device on first access, in the frame the view was made)
        or [] without appearance features."""
        if self._features is None:
            if not self.has_feature:
                self._features = []
            else:
                self._check_frame("features")
                self._features = [self._engine.read_feature(self._seq, self._slot)]
        return self._features

    @features.setter
    def features(self, v):
        self._features = v

    @property
    def mean(self):
        self._fetch()
        return self._mean

    @mean.setter
    def mean(self, v):
        self._mean = v

    @property
    def cov(self):
        self._fetch()
        return self._cov

    @cov.setter
    def cov(self, v):
        self._cov = v

    @property
    def kalman(self):
        return KALMAN_DICT[self.kalman_format]()


class BaseTracker(object):
    """SORT.  ``update`` == reference basetrack.py:368-487, executed by the fused kernel."""
    _kind = 'sort'

    def __init__(self, opts, frame_rate=30, *args, **kwargs):
        self.opts = opts
        self.frame_id = 0
        self.det_thresh = opts.conf_thresh
        self.buffer_size = int(frame_rate / 30.0 * opts.track_buffer)
        self.max_time_lost = self.buffer_size
        self.NMS = True
        self.kalman = KALMAN_DICT[self.opts.kalman_format]()
        if isinstance(opts.img_size, int):
            self.model_img_size = [opts.img_size, opts.img_size]
        elif isinstance(opts.img_size, (list, tuple)):
            self.model_img_size = opts.img_size
        self.debug_mode = False
        self._frame_rate = frame_rate
        self._engine = None
        # capacities of the device-side track pool (the reference has none): 1024 slots / 1024 detections per frame / 131072 candidate
        # pairs by default, opts.b2t_cap / b2t_dmax to change; an overflow raises B2TError (sticky) instead of dropping tracks silently
        self._engine_kw = dict(cap=int(getattr(opts, 'b2t_cap', 1024)), dmax=int(getattr(opts, 'b2t_dmax', 1024)),
                               dtype=getattr(opts, 'b2t_dtype', 'f64'))
        self._last = []
        self._removed = []
        self._watch_removed = False
        self._prev_lists = None

    # the reference exposes these three lists (basetrack.py:358-360); here they are views of the device-side lists
    @property
    def tracked_stracks(self):
        """Confirmed and unconfirmed Tracked-state tracks, in the reference's list order."""
        if self._engine is None or self.frame_id == 0:
            return []
        return self._views('tracked')

    @property
    def lost_stracks(self):
        if self._engine is None or self.frame_id == 0:
            return []
        return self._views('lost')

    @property
    def removed_stracks(self):
        """The tracks the reference passes to ``mark_removed``, appended in its order (see ``removed_in_step``).  The reference
        appends to this list forever; here the bookkeeping (three small device reads per frame) starts at the first access, so a
        caller that wants it from frame 1 reads the property once before tracking."""
        if not self._watch_removed:
            self._watch_removed = True
            self._prev_lists = self._read_lists()
        return list(self._removed)

    @removed_stracks.setter
    def removed_stracks(self, v):
        self._removed = list(v)

    def _read_lists(self):
        if self._engine is None or self.frame_id == 0:
            return {'tracked': np.zeros((0, 13)), 'lost': np.zeros((0, 13))}
        return {w: self._engine.read_list(0, w) for w in ('tracked', 'lost')}

    def _views(self, which):
        rows = self._engine.read_list(0, which)
        fmt = self.opts.kalman_format
        return [_TrackView(self._engine, 0, r, fmt, self.frame_id, extra=r[8:13]) for r in rows]

    def _get_engine(self, feat_dim=0):
        if self._engine is None:
            from b200track.engine import TrackEngine
            if self.opts.kalman_format == 'naive':
                raise NotImplementedError("kalman_format='naive' is not supported (see kalman_filter.NaiveKalmanFilter)")
            self._engine = TrackEngine(kind=self._kind, n_seq=1, kalman_format=self.opts.kalman_format,
                                       conf_thresh=self.opts.conf_thresh, iou_thresh=getattr(self.opts, 'iou_thresh', 0.5),
                                       track_buffer=self.opts.track_buffer, frame_rate=self._frame_rate,
                                       use_gmc=getattr(self, 'use_GMC', False), feat_dim=feat_dim, **self._engine_kw)
        if self._engine.feat_dim != feat_dim:
            raise RuntimeError("the tracker started with %s appearance features and now runs with %s: set use_apperance_model before "
                               "the first update" % (self._engine.feat_dim or "no", feat_dim or "none"))
        return self._engine

    @staticmethod
    def _to_numpy(det_results):
        if isinstance(det_results, torch.Tensor):
            det_results = det_results.detach().cpu().numpy()          # q14
        return np.ascontiguousarray(det_results, dtype=np.float32).reshape(-1, 6)

    def _warp(self, det_results, ori_img):
        return None

    def _step(self, det_results, ori_img, predict_only=False):
        if getattr(self, 'use_apperance_model', False):
            if self._kind != 'botsort':
                # ByteTrack's appearance mode (reference bytetrack.py:109-113) mixes gamma * IoU + (1 - gamma) * appearance into a DENSE
                # cost -- every track / detection pair becomes a candidate -- which the fused step's sparse assignment over
                # overlapping pairs cannot hold.  BoT-SORT's gated min(IoU, appearance) keeps the overlap structure and is built.
                raise NotImplementedError("use_apperance_model=True is built for BoTSORT only: %s's appearance cost is dense "
                                          "(gamma * IoU + (1 - gamma) * appearance over every pair) and needs another assignment path"
                                          % type(self).__name__)
            return self._finish_step(self._step_appearance(det_results, ori_img, predict_only), predict_only)
        eng = self._get_engine()
        self.frame_id += 1
        warp = None
        on_device = (not predict_only and isinstance(det_results, torch.Tensor) and det_results.is_cuda and det_results.device == eng.device
                     and type(self)._warp is BaseTracker._warp)
        if on_device:
            # the NMS output is already on the engine's device (tracker/track.py:151): boxes never visit the host
            rows = eng.step_cuda_dets([det_results.reshape(-1, 6)], id_base=[BaseTrack._count])[0]
        else:
            if not predict_only:
                dets = self._to_numpy(det_results)
                eng.load_dets([dets])
                warp = self._warp(dets, ori_img)
            rows = eng.step_host(warps=None if warp is None else np.asarray(warp, dtype=np.float64).reshape(1, 6),
                                 id_base=[BaseTrack._count], predict_only=predict_only)[0]
        return self._finish_step(rows, predict_only)

    def _finish_step(self, rows, predict_only=False):
        """Track views of the step's output rows; the id counter and the removed-list bookkeeping follow the engine."""
        eng = self._engine
        BaseTrack._count = int(eng.np_stat[0, L.STAT_NEXT_ID])
        rows = rows.copy()
        fmt = self.opts.kalman_format
        self._last = [_TrackView(eng, 0, rows[i], fmt, self.frame_id) for i in range(rows.shape[0])]
        if self._watch_removed:
            if not predict_only:                                   # update_without_detection removes nothing (basetrack.py:489-537)
                prev = self._prev_lists
                for r in removed_in_step(prev['tracked'], prev['lost'], eng.read_list(0, 'slots'), self.frame_id, self.max_time_lost):
                    self._removed.append(_TrackView(eng, 0, r, fmt, self.frame_id, extra=r[8:13]))
            self._prev_lists = self._read_lists()
        if self.debug_mode:
            print('===========Frame {}=========='.format(self.frame_id))
            print('Tracked: {}'.format([t.track_id for t in self._last]))
        return list(self._last)

    def update(self, det_results, ori_img):
        return self._step(det_results, ori_img)

    def update_without_detection(self, det_results, ori_img):
        return self._step(None, ori_img, predict_only=True)


def removed_in_step(prev_tracked, prev_lost, slots, frame_id, max_time_lost):
    """The rows of the tracks the reference appends to ``removed_stracks`` in one ``update``, in its order (basetrack.py:450-466,
    bytetrack.py:165-183): first the unconfirmed tracks the last association left unmatched, then every entry of the frame's OLD lost
    list that has gone more than ``max_time_lost`` frames without an update.  A track pruned in the previous frame is still in that
    list (the lost list is filtered against the removed list of the frame before), so unless it was re-found it is appended again.
    A track that ``remove_duplicate_stracks`` drops is not appended.
    prev_tracked / prev_lost: b2t_tracker_read_list rows at the end of the previous frame; slots: every slot's row after this
    frame's step (which = 2) -- a slot that left the lists keeps its state until a later frame's birth reuses it."""
    out = []
    for r in prev_tracked:
        s = slots[int(r[7])]
        if r[9] == 0 and s[8] == TrackState.Removed:
            out.append(s)
    for r in prev_lost:
        s = slots[int(r[7])]
        if frame_id - s[12] > max_time_lost:
            out.append(s)
    return out


def joint_stracks(tlista, tlistb):
    seen, res = set(), []
    for t in list(tlista) + list(tlistb):
        if t.track_id not in seen:
            seen.add(t.track_id)
            res.append(t)
    return res


def sub_stracks(tlista, tlistb):
    keep = OrderedDict()
    for t in tlista:
        keep[t.track_id] = t
    for t in tlistb:
        keep.pop(t.track_id, None)
    return list(keep.values())


def remove_duplicate_stracks(stracksa, stracksb):
    pdist = matching.iou_distance(stracksa, stracksb)
    dupa, dupb = set(), set()
    for p, q in zip(*np.where(pdist < 0.15)):
        if stracksa[p].frame_id - stracksa[p].start_frame > stracksb[q].frame_id - stracksb[q].start_frame:
            dupb.add(q)
        else:
            dupa.add(p)
    return ([t for i, t in enumerate(stracksa) if i not in dupa],
            [t for i, t in enumerate(stracksb) if i not in dupb])
