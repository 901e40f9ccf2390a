"""Per-frame access to tests/golden/loop_lifecycle.npz (written by tests/golden/make_golden_lifecycle.py): the reference trackers'
outputs, tracked / lost lists and removed-list appends on ``synth.lifecycle_stream`` streams, one entry per configuration.
NumPy only, shared by the oracle, host-simulator and GPU tiers."""
import os

import numpy as np

from b200track.synth import lifecycle_stream, stream_digest

PATH = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "loop_lifecycle.npz")
_npz = None


def load():
    global _npz
    if _npz is None:
        _npz = np.load(PATH, allow_pickle=False)
    return _npz


def configs():
    return [str(c) for c in load()["configs"]]


def _ragged(counts, values):
    off = np.concatenate([[0], np.cumsum(counts)])
    return [values[off[i]:off[i + 1]] for i in range(len(counts))]


class Config:
    """One configuration: ``frame(i)`` is the reference's state after frame i + 1."""

    def __init__(self, name):
        g = load()
        self.name = name
        self.kind, self.fmt = str(g[name + "_kind"]), str(g[name + "_fmt"])
        seed, n_obj, n_frames, conf, tb, fr, ws = g[name + "_params"]
        self.seed, self.n_obj, self.n_frames = int(seed), int(n_obj), int(n_frames)
        self.conf_thresh, self.track_buffer, self.frame_rate, self.warp_sigma = float(conf), int(tb), int(fr), float(ws)
        self.max_time_lost = int(self.frame_rate / 30.0 * self.track_buffer)
        self.digest = str(g[name + "_digest"])
        self.events = dict(zip([str(e) for e in g["events"]], g[name + "_events"].tolist()))
        self.out_ids = _ragged(g[name + "_out_n"], g[name + "_out_ids"])
        self.out_cls = _ragged(g[name + "_out_n"], g[name + "_out_cls"])
        self.rem_ids = _ragged(g[name + "_rem_n"], g[name + "_rem_ids"])
        self.rows = {w: _ragged(g[name + "_%s_n" % k], g[name + "_%s_rows" % k]) for w, k in (("tracked", "trk"), ("lost", "lost"))}
        self.tlwh_frames = [int(i) for i in g[name + "_tlwh_frames"]]
        self.tlwh = {}                                  # (which, frame) -> (n, 4) float64, which in out / tracked / lost
        for w, k in (("out", "out"), ("tracked", "trk"), ("lost", "lost")):
            counts = g[name + "_%s_n" % k][self.tlwh_frames]
            for i, v in zip(self.tlwh_frames, _ragged(counts, g[name + "_%s_tlwh" % k])):
                self.tlwh[(w, i)] = v

    def stream(self):
        frames, warps = lifecycle_stream(self.seed, self.n_frames, self.n_obj, conf_thresh=self.conf_thresh,
                                         warp_sigma=self.warp_sigma)
        assert stream_digest(frames) == self.digest, "lifecycle_stream drifted from the stream the golden was made from"
        return frames, (warps if self.kind == "botsort" else None)

    def oracle_kwargs(self):
        return dict(kind=self.kind, kalman_format=self.fmt, conf_thresh=self.conf_thresh, track_buffer=self.track_buffer,
                    frame_rate=self.frame_rate)

    def events_until(self, n_frames):
        """Prunings and duplicate drops visible in the first ``n_frames`` frames of the golden, counted from the stored lists: a
        pruned track is appended to removed_stracks while confirmed (is_activated); a duplicate drop is a track that leaves both
        lists without being appended."""
        prunes = dups = 0
        live, removed = {}, set()
        for i in range(n_frames):
            now = {int(r[0]): r for w in ("tracked", "lost") for r in self.rows[w][i]}
            appended = [int(t) for t in self.rem_ids[i]]
            for t in appended:
                if t in live and live[t][2] == 1 and t not in removed:
                    prunes += 1
            dups += sum(1 for t in live if t not in now and t not in removed and t not in appended)
            removed.update(appended)
            live = now
        return prunes, dups
