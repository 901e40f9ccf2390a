"""gpu: the body of track.py:132-179 with --tracker uavmot -- the tracker chosen from TRACKER_DICT among the drop-ins imported by their
bare names, update / update_without_detection, the per-frame result rows -- gives the reference's goldens, and the drop-in matching's
structure functions equal the oracle."""
import os
import sys

import numpy as np
import pytest

pytestmark = pytest.mark.gpu
torch = pytest.importorskip("torch")

HERE = os.path.dirname(os.path.abspath(__file__))
TRACKER = os.path.join(os.path.dirname(HERE), "yolov7-tracker_b200", "tracker")
sys.path.insert(0, HERE)
import uavmot_golden as UG                       # noqa: E402
import uavmot_oracle as U                        # noqa: E402

BARE = ("basetrack", "matching", "kalman_filter", "uavmot", "bytetrack", "botsort", "strongsort", "reid_models", "reid_models.OSNet",
        "reid_models.load_model_tools")


@pytest.fixture(scope="module")
def dropin():
    """the drop-in modules imported by their bare names, as track.py:16-23 does, and its TRACKER_DICT (track.py:55-63) over the
    trackers that have a drop-in"""
    saved = {k: sys.modules.pop(k) for k in list(sys.modules) if k in BARE}
    sys.path.insert(0, TRACKER)
    try:
        from basetrack import BaseTracker, BaseTrack
        from bytetrack import ByteTrack
        from botsort import BoTSORT
        from uavmot import UAVMOT, AMF_STrack
        from strongsort import StrongSORT
        import matching
        tracker_dict = {'sort': BaseTracker, 'bytetrack': ByteTrack, 'botsort': BoTSORT, 'uavmot': UAVMOT, 'strongsort': StrongSORT}
        yield tracker_dict, BaseTrack, AMF_STrack, matching
    finally:
        sys.path.remove(TRACKER)
        for k in BARE:
            sys.modules.pop(k, None)
        sys.modules.update(saved)


class _Opts:
    """track.py's argparse defaults that the body and the tracker read, with --tracker uavmot"""

    def __init__(self, fmt, track_buffer):
        self.tracker, self.gamma, self.detect_per_frame, self.min_area = "uavmot", 0.1, 1, 0.0
        self.conf_thresh, self.track_buffer, self.kalman_format, self.img_size = 0.2, track_buffer, fmt, 1280
        self.iou_thresh, self.reid_model_path, self.dhn_path = 0.5, "", ""


@pytest.mark.parametrize("name", [c.name for c in UG.CONFIGS])
def test_dropin_tracker_matches_reference(name, dropin):
    tracker_dict, BaseTrack, AMF_STrack, _ = dropin
    cfg = next(c for c in UG.CONFIGS if c.name == name).load()
    opts = _Opts(cfg.fmt, cfg.track_buffer)
    BaseTrack._count = 0
    tracker = tracker_dict[opts.tracker](opts, frame_rate=30, gamma=opts.gamma)          # track.py:132
    img0 = np.zeros((8, 8, 3), np.uint8)
    results = []
    for i, fr in enumerate(cfg.stream()):                                                  # track.py:138-179
        if not i % opts.detect_per_frame:
            out = torch.as_tensor(fr).cuda()                                               # post_process_v7's output, on the device
            current_tracks = tracker.update(out, img0)
        else:
            current_tracks = tracker.update_without_detection(None, img0)
        cur_tlwh, cur_id, cur_cls = [], [], []
        for trk in current_tracks:
            bbox, tid, cls = trk.tlwh, trk.track_id, trk.cls
            if bbox[2] * bbox[3] > opts.min_area:
                cur_tlwh.append(bbox)
                cur_id.append(tid)
                cur_cls.append(cls)
        results.append((i + 1, cur_id, cur_tlwh, cur_cls))
        assert cur_id == cfg.ids[i].tolist(), "frame %d" % (i + 1)
        np.testing.assert_allclose(np.array(cur_tlwh).reshape(-1, 4), cfg.tlwh[i], rtol=0, atol=1e-9)
    assert len(results) == cfg.n_frames
    assert isinstance(AMF_STrack(0, np.array([1, 2, 30, 40], np.float32), 0.9).get_xy(), np.ndarray)


class _T:
    def __init__(self, mean=None, xy=None):
        self.mean, self._xy = mean, xy

    def get_xy(self):
        return self._xy


def test_matching_structure_functions_match_oracle(dropin):
    matching = dropin[3]
    rng = np.random.default_rng(8)
    pts = np.concatenate([rng.integers(0, 8, (30, 2)) * 100.0, rng.uniform(0, 1280, (30, 2))])
    tracks = [_T(mean=np.r_[p + 0.25, np.zeros(6)]) for p in pts]
    dets = [_T(xy=p.astype(np.float32)) for p in pts[::-1]]
    a, b = U.structure_vectors(pts + 0.25), U.structure_vectors(pts[::-1].astype(np.float32), True)
    assert np.array_equal(matching.structure_representation(tracks), a)
    assert np.array_equal(matching.structure_representation(dets, mode="detection"), b)
    S = U.structure_distance(a, b)
    assert np.array_equal(matching.structure_similarity_distance(tracks, dets), S)
    cost = rng.uniform(0, 1, S.shape)
    assert np.array_equal(matching.local_relation_fuse_motion(cost, tracks, dets), 0.98 * cost + (1 - 0.98) * S)
    assert matching.structure_representation([]).shape == (0,)
