"""The configurations of tests/golden/loop_strongsort.npz (tests/golden/make_golden_strongsort.py) and their stored results.

TEST INFRASTRUCTURE.  Shared by the generator and by the oracle, host-simulator and GPU tests."""
import os

import numpy as np

from b200track.synth import make_strongsort_stream, stream_digest

PATH = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "loop_strongsort.npz")
FEAT_DIM = 64


class Config:
    """name, gamma, use_ECC, kalman_format, track_buffer, stream seed / objects / frames."""

    def __init__(self, name, gamma, use_ecc, fmt, track_buffer, seed, n_obj, n_frames):
        self.name, self.gamma, self.use_ecc, self.fmt, self.track_buffer = name, gamma, use_ecc, fmt, track_buffer
        self.seed, self.n_obj, self.n_frames = seed, n_obj, n_frames
        self.conf_thresh = 0.2
        self.max_time_lost = int(30 / 30.0 * track_buffer)

    def stream(self):
        """(frames, feats, warps): the warps are float32 values (stored as float64), as an ECC estimator returns them."""
        frames, feats, warps = make_strongsort_stream(self.seed, self.n_frames, self.n_obj, FEAT_DIM)
        return frames, feats, warps.astype(np.float32).astype(np.float64)

    def load(self):
        """Per-frame golden rows: ids, tlwh, lists {tracked, lost} (id, state, is_activated, start_frame, frame_id, tracklet_len),
        and {frame: features of the output tracks}."""
        z = np.load(PATH)
        p = self.name + "/"
        frames, feats, _ = self.stream()
        assert str(z[p + "digest"]) == stream_digest(frames) and str(z[p + "feat_digest"]) == stream_digest(feats), \
            "%s: the stream generator drifted from the golden" % self.name
        cnt = z[p + "count"]
        off = np.concatenate([[0], np.cumsum(cnt)])
        self.ids = [z[p + "ids"][off[i]:off[i + 1]] for i in range(self.n_frames)]
        self.tlwh = [z[p + "tlwh"][off[i]:off[i + 1]] for i in range(self.n_frames)]
        self.lists = {}
        for w in ("tracked", "lost"):
            c = z[p + w + "_count"]
            o = np.concatenate([[0], np.cumsum(c)])
            self.lists[w] = [z[p + w][o[i]:o[i + 1]] for i in range(self.n_frames)]
        fo = 0
        self.feats = {}
        for i in z[p + "feat_frames"]:
            n = cnt[i]
            self.feats[int(i)] = z[p + "feats"][fo:fo + n]
            fo += n
        return self


CONFIGS = [
    Config("default", 0.1, True, "strongsort", 30, 41, 40, 120),
    Config("nondefault", 0.3, False, "default", 6, 43, 40, 120),
]
