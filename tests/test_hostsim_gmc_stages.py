"""not-gpu: the ORB camera-motion stage checks of tests/gmc_stages.py on simulator builds of csrc/b2t_gmc.cu: more boxes over a row
than the row cache holds (with negative and out-of-frame corners), truncation at max_kp and matching on the truncated lists,
ds 1 / 3 / 4 at the 64-px minimum, reset(), the two-slot prepare / estimate_prepared form across a reset, several sequences with
none, some and no detections -- and builds with injected bugs failing at the stage they were made in."""
import ctypes as C
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "hostsim"))
import build_sim  # noqa: E402
import gmc_stages as GS  # noqa: E402
from simlib import ptr, sim  # noqa: E402
from b200track import _lib as L  # noqa: E402
from b200track import gmc as G  # noqa: E402
from b200track.synth import moved_frame, textured_frame  # noqa: E402

SYMBOLS = ["b2t_detect_last_error", "b2t_gmc_workspace_bytes", "b2t_gmc_workspace_layout", "b2t_gmc_reset", "b2t_gmc_estimate",
           "b2t_gmc_prepare", "b2t_gmc_estimate_prepared"]


class Sim:
    def __init__(self, lib, n_seq, h, w, ds=2, max_kp=4096):
        self.lib, self.S, self.h, self.w, self.ds, self.max_kp = lib, n_seq, h, w, ds, max_kp
        n = lib.b2t_gmc_workspace_bytes(n_seq, h, w, ds, max_kp)
        assert n > 0
        self.layout = G.workspace_layout(lib, n_seq, h, w, ds, max_kp)
        self.mem = np.zeros(n + 256, np.uint8)
        self.off = (-self.mem.ctypes.data) % 256
        self.ws = self.mem.ctypes.data + self.off
        self.warps = np.zeros((n_seq, 2, 3), np.float64)
        self.stat = np.zeros((n_seq, L.GMC_STAT_WORDS), np.int32)

    def _dets(self, dets, counts):
        return (0, None, None) if dets is None else (dets.shape[1], ptr(dets), ptr(counts))

    def estimate(self, frames, dets=None, counts=None, thresh=0.2):
        frames = np.ascontiguousarray(frames)
        dmax, dp, cp = self._dets(dets, counts)
        G.launch_estimate(self.lib, frames.ctypes.data, self.S, self.h, self.w, 3 * self.w, self.ds, dp, cp, dmax, thresh, self.ws, self.max_kp,
                          self.warps.ctypes.data, self.stat.ctypes.data, None)
        return self.warps.copy(), self.stat.copy()

    def prepare(self, frames, slot):
        frames = np.ascontiguousarray(frames)
        G._check(self.lib, self.lib.b2t_gmc_prepare(frames.ctypes.data, self.S, self.h, self.w, 3 * self.w, self.ds, self.ws, self.max_kp, slot, None))

    def estimate_prepared(self, slot, dets=None, counts=None, thresh=0.2):
        dmax, dp, cp = self._dets(dets, counts)
        G._check(self.lib, self.lib.b2t_gmc_estimate_prepared(self.S, self.h, self.w, self.ds, dp, cp, dmax, float(thresh), self.ws, self.max_kp, slot,
                                                              self.warps.ctypes.data, self.stat.ctypes.data, None))
        return self.warps.copy(), self.stat.copy()

    def reset(self):
        G._check(self.lib, self.lib.b2t_gmc_reset(self.ws, self.S, self.h, self.w, self.ds, self.max_kp, None))

    def bytes(self):
        return self.mem[self.off:].tobytes()


def run(est, seqs, dets=None, counts=None, thresh=0.2):
    """Every frame of seqs (n_seq lists of frames) through estimate, checked stage by stage.  Returns (failures, checker)."""
    ck = GS.Checker(est.S, est.ds, est.max_kp)
    md = [None] * est.S if dets is None else GS.thresholded(dets, counts, thresh)
    bad = []
    for k in range(len(seqs[0])):
        fr = np.stack([s[k] for s in seqs])
        warps, stat = est.estimate(fr, dets, counts, thresh)
        bad += [(k,) + b for b in ck.frame(fr, md, warps, stat, est.bytes(), est.layout)]
    return bad, ck


def moves(base, n=3):
    return [base] + [moved_frame(base, 0.2 * k, 1.5 * k, -1.0 * k) for k in range(1, n)]


def overflow_case():
    h, w = 160, 448
    base = textured_frame(31, h, w, n_rect=120)
    boxes = GS.many_boxes(h, w)
    dets = boxes[None].copy()
    return [moves(base)], dets, np.array([len(boxes)], np.int32)


def test_more_boxes_over_a_row_than_the_cache():
    seqs, dets, cnt = overflow_case()
    est = Sim(sim(), 1, 160, 448)
    bad, ck = run(est, seqs, dets, cnt)
    assert not bad, bad
    b = GS.many_boxes(160, 448)
    b = b[b[:, 4] >= np.float32(0.2)]
    y = 80 // 2                                                            # a working row every tall box covers
    assert (((b[:, 1] / 2).astype(int) <= y) & ((b[:, 3] / 2).astype(int) > y)).sum() > 256
    ky = np.concatenate([GS.OG.GMCOracle().stages(f, b)[2] for f in seqs[0]])
    assert ((ky >= 0.3 * 80) & (ky < 0.7 * 80)).sum() > 20                   # corners survive on the overflowing rows


def truncation_case():
    base = textured_frame(32, 200, 300, n_rect=150)
    return [moves(base)]


def test_truncation_at_max_kp_and_matching_on_the_truncated_lists():
    est = Sim(sim(), 1, 200, 300, max_kp=64)
    bad, _ = run(est, truncation_case())
    assert not bad, bad
    assert est.stat[0, 5] & L.GMC_TRUNCATED and est.stat[0, 0] == 64


@pytest.mark.parametrize("ds", [1, 3, 4])
def test_other_downscales_at_the_64px_minimum(ds):
    for h, w in ((64 * ds, 64 * ds), (64 * ds + ds - 1, 96 * ds + 1)):
        base = textured_frame(33 + ds, h, w, n_rect=40)
        bad, _ = run(Sim(sim(), 1, h, w, ds=ds), [moves(base)])
        assert not bad, (ds, h, w, bad)
    assert sim().b2t_gmc_workspace_bytes(1, 63 * ds, 200 * ds, ds, 4096) == 0


def test_sequences_with_none_some_and_no_detections_and_reset():
    h, w = 128, 192
    seqs = [moves(textured_frame(40 + s, h, w, n_rect=80)) for s in range(3)]
    dets = np.zeros((3, 8, 6), np.float32)
    dets[1, :3] = [[10, 10, 60, 90, 0.9, 0], [100, 40, 150, 120, 0.5, 0], [120, 0, 190, 50, 0.1, 0]]
    dets[2, :8] = np.concatenate([GS.many_boxes(h, w, 5, seed=2)[:8]])[:8]
    counts = np.array([0, 3, 8], np.int32)
    est = Sim(sim(), 3, h, w)
    bad, _ = run(est, seqs, dets, counts)
    assert not bad, bad
    bad, _ = run(Sim(sim(), 3, h, w), seqs)                              # dets=None
    assert not bad, bad
    est.reset()
    warps, stat = est.estimate(np.stack([s[2] for s in seqs]), dets, counts, 0.2)
    assert (stat[:, 5] & L.GMC_FIRST_FRAME).all() and np.array_equal(warps, np.tile(np.eye(2, 3), (3, 1, 1)))


def test_prepared_slots_across_a_reset_equal_estimate():
    h, w = 128, 192
    seqs = [moves(textured_frame(50 + s, h, w, n_rect=80), 4) for s in range(2)]
    a, b = Sim(sim(), 2, h, w), Sim(sim(), 2, h, w)
    slot = 0
    for k in list(range(4)) + ["reset"] + list(range(3)):
        if k == "reset":
            a.reset(); b.reset()
            continue
        fr = np.stack([s[k] for s in seqs])
        w1, s1 = a.estimate(fr)
        b.prepare(fr, slot)
        w2, s2 = b.estimate_prepared(slot)
        slot ^= 1
        assert np.array_equal(w1, w2) and np.array_equal(s1, s2), k


# ---------------------------------------------------------------------------------------------- injected bugs
GMC = "b2t_gmc.cu"
BUGS = {
    # name: (patches, the stage the harness must fail at, the case)
    "overflow_box_test_skipped": ([(GMC, "if (x >= bx0 && x < bx1 && y >= by0 && y < by1) keep = false;", "(void)bx0; (void)bx1; (void)by0; (void)by1;")],
                                  "keypoints", "overflow"),
    "second_best_dropped": ([(GMC, "else if (d < d2) d2 = d;", "")], "ratio", "truncation"),
    "truncated_flag_not_set": ([(GMC, "if (state[3]) flags |= B2T_GMC_TRUNCATED;", "")], "flags", "truncation"),
}


@pytest.mark.parametrize("bug", sorted(BUGS))
def test_injected_bug_fails_at_its_stage(bug):
    patches, stage, case = BUGS[bug]
    lib = L.declare(C.CDLL(build_sim.build_variant("gmc_" + bug, patches, units=(GMC, "b2t_nms.cu"))), names=SYMBOLS)
    if case == "overflow":
        seqs, dets, cnt = overflow_case()
        bad, _ = run(Sim(lib, 1, 160, 448), seqs, dets, cnt)
    else:
        bad, _ = run(Sim(lib, 1, 200, 300, max_kp=64), truncation_case())
    print(bug, bad[:3])
    assert bad and bad[0][2] == stage, bad
