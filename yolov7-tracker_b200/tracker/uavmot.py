"""Drop-in for the reference's ``tracker/uavmot.py``: ``UAVMOT(opts, frame_rate=30, gamma=0.1)`` with
``update(det_results, ori_img) -> List[STrack]`` (reference :106-279), executed as one fused kernel per frame (csrc/b2t_step.cuh,
kind = uavmot): ByteTrack's stages, association 1 re-solved on the structure-fused cost when its IoU solve matched (q20), and the
wrong-track marking of association 2 (q21).  The appearance branch is unreachable in the reference (``use_apperance_model = False``,
:76), so the ReID extractor is not loaded."""
import _b2t_path  # noqa: F401
from basetrack import TrackState, STrack, BaseTracker, joint_stracks, sub_stracks, remove_duplicate_stracks  # noqa: F401


class AMF_STrack(STrack):
    """The reference's track type (:14-69), for code that builds or inspects tracks directly; the tracker itself keeps its tracks on
    the device."""

    def __init__(self, cls, tlwh, score, kalman_format='default', feature=None) -> None:
        super().__init__(cls, tlwh, score, kalman_format, feature)

    def AMF_update(self, new_track, frame_id):
        self.frame_id = frame_id
        self.tracklet_len += 1
        self.mean, self.cov = None, None
        self._tlwh[:4] = new_track.tlwh[:4]
        self.mean, self.cov = self.kalman.initiate(self._measure(self._tlwh))
        self.state = TrackState.Tracked
        self.is_activated = True
        self.score = new_track.score

    def AMF_reactivate(self, new_track, frame_id, new_id=False):
        self.mean, self.cov = self.kalman.initiate(self._measure(new_track.tlwh))
        self.tracklet_len = 0
        self.state = TrackState.Tracked
        self.is_activated = True
        self.frame_id = frame_id
        if new_id:
            self.track_id = self.next_id()
        self.score = new_track.score

    def get_xy(self):
        """centre as structure_representation reads it: tlwh2xywh(tlwh)[:2] = tl + wh // 2"""
        return self.tlwh2xywh(self.tlwh)[:2]


class UAVMOT(BaseTracker):
    _kind = 'uavmot'

    def __init__(self, opts, frame_rate=30, gamma=0.1, *args, **kwargs):
        super().__init__(opts, frame_rate, *args, **kwargs)
        self.use_apperance_model = False
        self.reid_model = None
        self.gamma = gamma
        self.low_conf_thresh = max(0.15, self.opts.conf_thresh - 0.3)
        self.filter_small_area = False
