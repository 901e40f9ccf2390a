"""-m gpu: the ORB camera-motion estimator (csrc/b2t_gmc.cu) stage by stage on an H100 with tests/gmc_stages.py: key points and
descriptors bit for bit, the ratio / sigma point set, RANSAC's best hypothesis exactly and the fit within a derived bound -- at the
benchmark geometry (8 x 1280^2, ~300 boxes, max_kp 32768), with more boxes over a row than the row cache holds, under truncation,
at ds 1 / 3 / 4 and the 64-px minimum, across reset(), in the two-slot prepare / estimate_prepared form and with sequences that have
none, some and no detections."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu
torch = pytest.importorskip("torch")

import gmc_stages as GS  # noqa: E402
from b200track import _lib as L  # noqa: E402
from b200track.gmc import GmcEstimator  # noqa: E402
from b200track.synth import make_stream, moved_frame, pack_frames, textured_frame  # noqa: E402


class Dev:
    """GmcEstimator with host arrays in and out (the interface of the simulator tier's runner)."""

    def __init__(self, n_seq, h, w, ds=2, max_kp=4096):
        self.e = GmcEstimator(n_seq, h, w, ds, max_kp=max_kp)
        self.S, self.ds, self.max_kp, self.layout = n_seq, ds, max_kp, self.e.layout

    @staticmethod
    def _d(a):
        return None if a is None else torch.from_numpy(np.ascontiguousarray(a)).cuda()

    def estimate(self, frames, dets=None, counts=None, thresh=0.2):
        w, s = self.e.estimate(self._d(frames), self._d(dets), self._d(counts), thresh)
        return w.cpu().numpy(), s.cpu().numpy()

    def prepare(self, frames, slot):
        self.e.prepare(self._d(frames), slot)

    def estimate_prepared(self, slot, dets=None, counts=None, thresh=0.2):
        w, s = self.e.estimate_prepared(slot, self._d(dets), self._d(counts), thresh)
        return w.cpu().numpy(), s.cpu().numpy()

    def reset(self):
        self.e.reset()

    def bytes(self):
        return self.e.ws.cpu().numpy().tobytes()


def run(est, seqs, dets=None, counts=None, thresh=0.2):
    ck = GS.Checker(est.S, est.ds, est.max_kp)
    md = [None] * est.S if dets is None else GS.thresholded(dets, counts, thresh)
    bad = []
    for k in range(len(seqs[0])):
        fr = np.stack([s[k] for s in seqs])
        warps, stat = est.estimate(fr, dets, counts, thresh)
        bad += [(k,) + b for b in ck.frame(fr, md, warps, stat, est.bytes(), est.layout)]
    print(ck.report)
    return bad, ck


def moves(base, n=3):
    return [base] + [moved_frame(base, 0.2 * k, 1.5 * k, -1.0 * k) for k in range(1, n)]


def test_benchmark_geometry():
    """8 x 1280^2 frames moved by known shifts, ~300 boxes per frame at det_thresh 0.2, max_kp 32768 (bench_sub.gmc_estimation)."""
    n, size = 8, 1280
    base = [textured_frame(7000 + s, size, size, n_rect=1500) for s in range(n)]
    seqs = [[b, np.ascontiguousarray(np.roll(b, (3, -2), (0, 1)))] for b in base]
    dets, cnt = pack_frames(make_stream(7100, n, 300, img=size)[0], 320)
    bad, ck = run(Dev(n, size, size, 2, 32768), seqs, dets, cnt)
    assert not bad, bad
    assert ck.report["points"] > 1000


def test_more_boxes_over_a_row_than_the_cache():
    h, w = 320, 896
    boxes = GS.many_boxes(h, w)
    bad, _ = run(Dev(1, h, w), [moves(textured_frame(31, h, w, n_rect=300))], boxes[None].copy(), np.array([len(boxes)], np.int32))
    assert not bad, bad


def test_truncation_at_max_kp():
    est = Dev(1, 400, 600, max_kp=64)
    bad, _ = run(est, [moves(textured_frame(32, 400, 600, n_rect=300))])
    assert not bad, bad


@pytest.mark.parametrize("ds", [1, 3, 4])
def test_other_downscales_at_the_64px_minimum(ds):
    for h, w in ((64 * ds, 64 * ds), (64 * ds + ds - 1, 96 * ds + 1), (360 * ds // 2, 640 * ds // 2)):
        bad, _ = run(Dev(1, h, w, ds=ds), [moves(textured_frame(33 + ds, h, w, n_rect=60))])
        assert not bad, (ds, h, w, bad)


def test_eight_sequences_none_some_and_no_detections_then_reset():
    h, w = 360, 640
    seqs = [moves(textured_frame(40 + s, h, w, n_rect=200)) for s in range(8)]
    dets = np.zeros((8, 64, 6), np.float32)
    counts = np.array([0, 3, 64, 0, 10, 1, 40, 64], np.int32)
    for s in range(8):
        dets[s, :counts[s]] = GS.many_boxes(h, w, 64, seed=s)[:counts[s]]
    est = Dev(8, h, w)
    bad, _ = run(est, seqs, dets, counts)
    assert not bad, bad
    bad, _ = run(Dev(8, h, w), seqs)
    assert not bad, bad
    est.reset()
    warps, stat = est.estimate(np.stack([s[2] for s in seqs]), dets, counts)
    assert (stat[:, 5] & L.GMC_FIRST_FRAME).all() and np.array_equal(warps, np.tile(np.eye(2, 3), (8, 1, 1)))


def test_prepared_slots_across_a_reset_equal_estimate():
    h, w = 360, 640
    seqs = [moves(textured_frame(50 + s, h, w, n_rect=200), 4) for s in range(2)]
    a, b = Dev(2, h, w), Dev(2, h, w)
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
