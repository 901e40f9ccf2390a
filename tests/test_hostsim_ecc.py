"""not-gpu: csrc/b2t_ecc.cu executed by the fiber simulator (library built by tests/hostsim/build_sim_ecc.py; one block at a time, so
the iteration kernel runs with a cluster of one CTA; the distributed-shared-memory combine of the GPU build is covered by tests/test_gpu_ecc.py) against the cv2 fixtures of
tests/golden/ecc.npz and against oracle/ecc.py: the preparation bit for bit, the warp stage bit for bit, and the loop iteration by
iteration (rho and map)."""
import ctypes as C
import os
import sys

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "hostsim"))
sys.path.insert(0, os.path.join(HERE, "golden"))
from build_sim_ecc import sim_ecc  # noqa: E402
from b200track import _lib as L  # noqa: E402
from b200track import gmc as G  # noqa: E402
from b200track.synth import textured_frame  # noqa: E402
from make_golden_ecc import CASES, SMALL, WARP_MAPS, frames, plane_digest, warp_plane  # noqa: E402
from oracle import ecc as E  # noqa: E402

GOLD = np.load(os.path.join(HERE, "golden", "ecc.npz"))


def lib():
    return sim_ecc()


class SimEcc:
    def __init__(self, n_seq, h, w, ds=2):
        self.lib = lib()
        self.S, self.h, self.w, self.ds = n_seq, h, w, ds
        n = self.lib.b2t_ecc_workspace_bytes(n_seq, h, w, ds)
        assert n > 0
        self.layout = G.ecc_workspace_layout(self.lib, n_seq, h, w, ds)
        self.mem = np.zeros(n + 256, np.uint8)
        self.off = (-self.mem.ctypes.data) % 256
        self.warps = np.zeros((n_seq, 2, 3), np.float64)
        self.stat = np.zeros((n_seq, L.GMC_STAT_WORDS), np.int32)

    def reset(self):
        G._check(self.lib, self.lib.b2t_ecc_reset(self.mem.ctypes.data + self.off, self.S, self.h, self.w, self.ds, None))

    def estimate(self, frames, max_iter=100, eps=1e-5):
        frames = np.ascontiguousarray(frames)
        G.launch_ecc(self.lib, frames.ctypes.data, self.S, self.h, self.w, 3 * self.w, self.ds, max_iter, eps, self.mem.ctypes.data + self.off,
                     self.warps.ctypes.data, self.stat.ctypes.data, None)
        return self.warps.copy(), self.stat.copy()

    def plane(self, seq, which):
        o = self.off + seq * self.layout["stride"] + self.layout[which]
        return self.mem[o:o + self.layout["h"] * self.layout["w"]].reshape(self.layout["h"], self.layout["w"]).copy()


@pytest.mark.parametrize("k", [1, 3, 5])
def test_prepare_bit_exact_with_cv2_planes(k):
    case = CASES[k]
    fr = frames(case)
    e = SimEcc(1, case["h"], case["w"])
    e.estimate(fr[0][None], max_iter=1)
    t0 = e.plane(0, "template")
    assert np.array_equal(plane_digest(t0), GOLD["plane_sha%d" % k][0])
    e.estimate(fr[1][None], max_iter=1)
    assert np.array_equal(plane_digest(e.plane(0, "current")), GOLD["plane_sha%d" % k][1])
    assert np.array_equal(e.plane(0, "template"), t0)                                # the template stays the first frame (q17)
    if k in SMALL:
        assert np.array_equal(t0, GOLD["plane%d" % k][0]) and np.array_equal(e.plane(0, "current"), GOLD["plane%d" % k][1])


def test_prepare_other_downscales_equal_oracle():
    f = textured_frame(3, 75, 97, n_rect=40)
    for ds in (1, 3):
        e = SimEcc(1, 75, 97, ds)
        e.estimate(f[None], max_iter=1)
        assert np.array_equal(e.plane(0, "template"), E.prepare(f, ds)), ds


def test_warp_stage_bit_exact_with_cv2_warpaffine():
    P = np.ascontiguousarray(warp_plane())
    h, w = P.shape
    lb = lib()
    for j in range(len(WARP_MAPS)):
        M = np.ascontiguousarray(GOLD["warp_maps"][j].reshape(6), np.float32)
        img, gx, gy = (np.zeros((h, w), np.float32) for _ in range(3))
        mask = np.zeros((h, w), np.uint8)
        G._check(lb, lb.b2t_ecc_warp(P.ctypes.data, h, w, M.ctypes.data_as(C.POINTER(C.c_float)), img.ctypes.data, gx.ctypes.data, gy.ctypes.data,
                                     mask.ctypes.data, None))
        assert np.array_equal(img, GOLD["warp_img"][j]) and np.array_equal(gx, GOLD["warp_gx"][j]) and np.array_equal(gy, GOLD["warp_gy"][j]), j
        assert np.array_equal(mask, GOLD["warp_mask"][j]), j


def _loop_vs_oracle(f0, f1, n_check):
    h, w = f0.shape[:2]
    t, im = E.prepare(f0), E.prepare(f1)
    trace = []
    Hf, it, fl, rho = E.ecc(t, im, trace=trace)
    e = SimEcc(1, h, w)
    for k in range(1, min(n_check, it) + 1):
        e.reset()
        e.estimate(f0[None])
        warps, stat = e.estimate(f1[None], max_iter=k)
        assert stat[0, 0] == k and stat[0, 7] == 1
        if k <= len(trace):
            r, Mk = trace[k - 1]
            assert abs(G.ecc_rho(stat)[0] - r) < 1e-9, (k, G.ecc_rho(stat)[0], r)
            np.testing.assert_allclose(warps[0], Mk, rtol=0, atol=1e-6, err_msg="iteration %d" % k)
    e.reset()
    e.estimate(f0[None])
    warps, stat = e.estimate(f1[None])
    assert stat[0, 0] == it and stat[0, 5] == fl
    np.testing.assert_allclose(warps[0], Hf, rtol=0, atol=1e-6)
    assert warps.dtype == np.float64 and np.array_equal(warps[0], warps[0].astype(np.float32))
    return it, fl


def test_loop_per_iteration_equals_oracle_converging():
    from b200track.synth import moved_frame
    base = textured_frame(7, 120, 160, n_rect=60)
    it, fl = _loop_vs_oracle(base, moved_frame(base, 0.3, 1, -1), 12)               # rotation + shift: 11 iterations
    assert fl == E.CONVERGED and it > 2


def test_loop_iteration_cap_equals_oracle():
    base = textured_frame(7, 120, 160, n_rect=60)
    it, fl = _loop_vs_oracle(base, np.ascontiguousarray(np.roll(base, (2, -3), (0, 1))), 4)    # the wrapped roll oscillates
    assert fl == E.ITER_CAP and it == 100


def test_loop_failure_keeps_last_map_and_flags():
    case = CASES[5]                                            # lambda_d <= 0 after two completed updates
    fr = frames(case)
    it, fl = _loop_vs_oracle(fr[0], fr[1], 3)
    assert fl == E.FAILED_LAMBDA and it == GOLD["it5"][1]
    case = CASES[3]                                            # flat frame: identity
    fr = frames(case)
    e = SimEcc(1, case["h"], case["w"])
    e.estimate(fr[0][None])
    warps, stat = e.estimate(fr[1][None])
    assert stat[0, 5] == E.FAILED_LAMBDA and stat[0, 0] == 1 and np.array_equal(warps[0], np.eye(2, 3))


def test_first_frame_reset_and_bad_geometry():
    f = textured_frame(8, 64, 80, n_rect=30)
    e = SimEcc(2, 64, 80)
    warps, stat = e.estimate(np.stack([f, f]))
    assert np.array_equal(warps, np.tile(np.eye(2, 3), (2, 1, 1))) and (stat[:, 5] == E.FIRST_FRAME).all() and (stat[:, 0] == 0).all()
    warps, stat = e.estimate(np.stack([f, f]))
    assert (stat[:, 5] == E.CONVERGED).all() and (stat[:, 7] == 1).all() and np.abs(warps - np.eye(2, 3)).max() < 1e-6
    e.reset()
    _, stat = e.estimate(np.stack([f, f]))
    assert (stat[:, 5] == E.FIRST_FRAME).all()
    lb = lib()
    assert lb.b2t_ecc_workspace_bytes(1, 14, 100, 2) == 0                        # 7 working rows: below the 8 x 8 minimum
    assert lb.b2t_ecc_estimate(None, 1, 64, 80, 240, 2, 100, 1e-5, None, None, None, None) != 0
    assert lb.b2t_ecc_estimate(f.ctypes.data, 1, 64, 80, 240, 2, 0, 1e-5, e.mem.ctypes.data + e.off, e.warps.ctypes.data, None, None) != 0
