"""The stream and configurations of tests/golden/loop_uavmot.npz (tests/golden/make_golden_uavmot.py) and their stored results.

TEST INFRASTRUCTURE.  Shared by the generator and by the oracle, host-simulator and GPU tests.

The stream is built so that UAVMOT's structure term and quirks all act (a random stream almost never lets S decide a match):
  * a lattice of objects 100 px apart, each drifting by its own fraction of a pixel per frame: their detection centres are integers
    near the lattice, so the neighbour lengths tie (maximum and minimum), some lie exactly on 400 and some just inside it, and the
    offsets include axis and diagonal directions;
  * an isolated object (> 400 px from everything) and a pair of objects that only see each other;
  * duplicate detections of some objects, shifted by a few pixels with score 0.25 (high, never born), which compete with the
    object's own detection in the fused solve; on a few frames per configuration a duplicate is placed (``placed``) so that the two
    IoU distances differ by less than the structure term moves them and S decides which one the track takes (a random stream
    almost never has such a frame);
  * low-score detections, misses and re-appearances (association 2, q21, re-activation);
  * each box jitters by a pixel, so that the tracks' Kalman centres do not move as exact translations of each other;
  * frame 2 has two detections: the first track's own, and the second object's shifted by 25 px (IoU distance ~0.76, above 0.7 and
    below 0.8): association 1's only match is (0, 0), q20 skips the fused solve, and the second track goes unmatched."""
import hashlib
import os

import numpy as np

PATH = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "loop_uavmot.npz")


def make_uavmot_stream(seed, n_frames=60, skip_frame=2, placed=()):
    """placed: ((frame, object, dx, dy, dw, dh), ...) -- duplicates put where S decides association 1 (found by
    tests/golden/make_golden_uavmot.py's search); the random duplicates keep their draws, so a placement leaves earlier frames as
    they were"""
    rng = np.random.default_rng(seed)
    placed = {(p[0], p[1]): p[2:] for p in placed}
    objs = []                                    # (cx, cy, w, h, vx, vy)
    for gy in range(4):
        for gx in range(5):
            objs.append([300 + 100 * gx, 250 + 100 * gy, 40 + 2 * ((gx + gy) % 3), 80 + 4 * (gx % 2), 2, 1])
    objs.append([1150, 1150, 50, 90, -1, -1])    # isolated
    objs.append([150, 1000, 44, 88, 1, -1])      # a pair that only sees each other
    objs.append([150, 1100, 46, 84, 1, -1])
    objs.append([300 + 400, 250 + 300 + 400 - 1, 42, 80, 2, 1])   # just inside 400 of the lattice corner
    objs = np.array(objs, np.float64)
    n = len(objs)
    # each object drifts by its own fraction of a pixel per frame: the detection centres stay integers near the lattice (ties, 400,
    # axes and diagonals come and go), while the tracks' Kalman centres keep generic offsets (no length or angle near a tie)
    objs[:, 4:6] += rng.uniform(-0.3, 0.3, (n, 2))
    frames = []
    for f in range(1, n_frames + 1):
        rows = []
        for k in range(n):
            cx, cy, w, h, vx, vy = objs[k]
            x, y = cx + vx * f, cy + vy * f
            miss = (k % 7 == 3 and 12 <= f < 16) or (k % 9 == 5 and 25 <= f < 27)
            if f == skip_frame and k > 1:
                continue
            if miss:
                continue
            x1, y1 = round(x - w / 2) + int(rng.integers(-1, 2)), round(y - h / 2) + int(rng.integers(-1, 2))
            if f == skip_frame and k == 1:
                x1 += 25             # IoU distance ~0.76 to its track: matchable only by the fused solve at 0.8, which q20 skips
            score = 0.9 if not (k % 5 == 2 and f % 6 == 0) else 0.17       # low rows now and then (association 2)
            rows.append([x1, y1, x1 + w, y1 + h, score, k % 3])
            dup = None
            if f != skip_frame and f > 3 and k < 20 and (f + k) % 4 == 0:
                # a duplicate a few pixels off, high but below the birth threshold
                dup = (int(rng.integers(-6, 7)), int(rng.integers(-6, 7)), int(rng.integers(-3, 4)), int(rng.integers(-3, 4)))
            dup = placed.get((f, k), dup)
            if dup is not None:
                dx, dy, dw, dh = dup
                rows.append([x1 + dx, y1 + dy, x1 + dx + w + dw, y1 + dy + h + dh, 0.25, k % 3])
        a = np.array(rows, np.float32).reshape(-1, 6)
        frames.append(a)
    return frames


def stream_digest(frames):
    h = hashlib.sha1()
    for a in frames:
        h.update(np.ascontiguousarray(a, np.float32).tobytes())
    return h.hexdigest()


class Config:
    def __init__(self, name, fmt, track_buffer, seed, n_frames, placed=()):
        self.name, self.fmt, self.track_buffer, self.seed, self.n_frames = name, fmt, track_buffer, seed, n_frames
        self.placed = tuple(placed)
        self.conf_thresh = 0.2

    def stream(self):
        return make_uavmot_stream(self.seed, self.n_frames, placed=self.placed)

    def load(self):
        z = np.load(PATH)
        p = self.name + "/"
        frames = self.stream()
        assert str(z[p + "digest"]) == stream_digest(frames), "%s: the stream generator drifted from the golden" % self.name
        cnt = z[p + "count"]
        off = np.concatenate([[0], np.cumsum(cnt)])
        self.ids = [z[p + "ids"][off[i]:off[i + 1]] for i in range(self.n_frames)]
        self.tlwh = [z[p + "tlwh"][off[i]:off[i + 1]] for i in range(self.n_frames)]
        self.lists = {}
        for w in ("tracked", "lost"):
            c = z[p + w + "_count"]
            o = np.concatenate([[0], np.cumsum(c)])
            self.lists[w] = [z[p + w][o[i]:o[i + 1]] for i in range(self.n_frames)]
        return self


CONFIGS = [
    Config("default", "default", 30, 12, 60, placed=[(10, 11, 0, -4, 1, 0)]),
    Config("botsort_short", "botsort", 5, 14, 60, placed=[(12, 11, 2, 0, -1, -1), (30, 4, 0, 1, 2, -2)]),
]
