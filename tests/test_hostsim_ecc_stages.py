"""not-gpu: the ECC stage harnesses of tests/ecc_stages.py on simulator builds of csrc/b2t_ecc.cu (cluster of one CTA, the host's
libm): the warp stage on the edge maps and planes bit for bit, the preparation at ds 1 - 5, every iteration from the kernel's own
previous map within ``ecc_step_ref``'s bound, and builds with injected bugs failing at the stage or iteration they were made in."""
import ctypes as C
import os
import sys

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "hostsim"))
sys.path.insert(0, os.path.join(HERE, "golden"))
import build_sim  # noqa: E402
import ecc_stages as ES  # noqa: E402
from build_sim_ecc import SYMBOLS, sim_ecc  # noqa: E402
from b200track import _lib as L  # noqa: E402
from b200track import gmc as G  # noqa: E402
from b200track.synth import moved_frame, textured_frame  # noqa: E402
from make_golden_ecc import CASES, frames  # noqa: E402
from oracle import ecc as E  # noqa: E402


class Sim:
    """n sequences of (h, w) frames on a simulator library: reset, the first frames as templates, then the second frames."""

    def __init__(self, lib, h, w, ds=2, n_seq=1):
        self.lib, self.h, self.w, self.ds, self.S = lib, h, w, ds, n_seq
        n = lib.b2t_ecc_workspace_bytes(n_seq, h, w, ds)
        assert n > 0
        self.layout = G.ecc_workspace_layout(lib, n_seq, h, w, ds)
        self.mem = np.zeros(n + 256, np.uint8)
        self.ws = self.mem.ctypes.data + (-self.mem.ctypes.data) % 256
        self.warps = np.zeros((n_seq, 2, 3), np.float64)
        self.stat = np.zeros((n_seq, L.GMC_STAT_WORDS), np.int32)

    def estimate(self, fr, max_iter=100):
        fr = np.ascontiguousarray(fr)
        G.launch_ecc(self.lib, fr.ctypes.data, self.S, self.h, self.w, 3 * self.w, self.ds, max_iter, 1e-5, self.ws, self.warps.ctypes.data,
                     self.stat.ctypes.data, None)
        return self.warps.copy(), self.stat.copy()

    def pair(self, f0, f1, max_iter):
        G._check(self.lib, self.lib.b2t_ecc_reset(self.ws, self.S, self.h, self.w, self.ds, None))
        self.estimate(f0)
        return self.estimate(f1, max_iter)

    def plane(self, seq, which):
        o = self.ws - self.mem.ctypes.data + seq * self.layout["stride"] + self.layout[which]
        return self.mem[o:o + self.layout["h"] * self.layout["w"]].reshape(self.layout["h"], self.layout["w"]).copy()


def sim_warp(lib):
    def warp(P, M):
        P = np.ascontiguousarray(P)
        h, w = P.shape
        out = [np.zeros((h, w), np.float32) for _ in range(3)] + [np.zeros((h, w), np.uint8)]
        Mh = np.ascontiguousarray(np.asarray(M, np.float32).reshape(6))
        G._check(lib, lib.b2t_ecc_warp(P.ctypes.data, h, w, Mh.ctypes.data_as(C.POINTER(C.c_float)), *[o.ctypes.data for o in out], None))
        return out
    return warp


# ---------------------------------------------------------------------------------------------- cases (small: the simulator is slow)
def converging():
    base = textured_frame(7, 120, 160, n_rect=60)
    return base, moved_frame(base, 0.3, 1, -1)


def rolling():
    base = textured_frame(7, 120, 160, n_rect=60)
    return base, np.ascontiguousarray(np.roll(base, (2, -3), (0, 1)))


def lambda_failure():
    return tuple(frames(CASES[5]))


ITER_CASES = {"converging": (converging, 12), "roll": (rolling, 10), "lambda": (lambda_failure, 4)}


def run_iterate(lib, pairs, K):
    h, w = pairs[0][0].shape[:2]
    sim = Sim(lib, h, w, n_seq=len(pairs))
    f0, f1 = np.stack([p[0] for p in pairs]), np.stack([p[1] for p in pairs])
    planes = [ES.ecc_planes(a, b) for a, b in pairs]
    return ES.iterate(lambda k: sim.pair(f0, f1, k), planes, K, cluster=1, device=False)


def warp_failures(lib, shapes=((8, 8), (31, 47))):
    warp = sim_warp(lib)
    bad = []
    for h, w in shapes:
        P = ES.edge_plane(h, w)
        for name, M in ES.EDGE_MAPS:
            if ES.warp_mismatches(warp, P, M):
                bad.append((h, w, name))
    return bad


# ---------------------------------------------------------------------------------------------- the shipped source
@pytest.mark.parametrize("shape", [(2, 2), (8, 8), (31, 47), (397, 403)])
def test_warp_edge_maps_bit_exact(shape):
    warp = sim_warp(sim_ecc())
    P = ES.edge_plane(*shape)
    for name, M in ES.EDGE_MAPS:
        assert ES.warp_mismatches(warp, P, M) == [], name


@pytest.mark.parametrize("ds", [1, 2, 3, 4, 5])
def test_prepare_every_downscale(ds):
    for h, w in ((8 * ds, 8 * ds), (8 * ds + 1, 8 * ds + ds - 1 if ds > 1 else 9), (57, 83)):
        rng = np.random.default_rng(ds * 1000 + h * 7 + w)
        fa, fb = (rng.integers(0, 256, (h, w, 3), dtype=np.uint8) for _ in range(2))
        sim = Sim(sim_ecc(), h, w, ds)
        sim.pair(fa, fb, 1)
        assert np.array_equal(sim.plane(0, "template"), E.prepare(fa, ds)), (ds, h, w)
        assert np.array_equal(sim.plane(0, "current"), E.prepare(fb, ds)), (ds, h, w)


@pytest.mark.parametrize("case", sorted(ITER_CASES))
def test_every_iteration_from_its_own_previous_map(case):
    make, K = ITER_CASES[case]
    rep = run_iterate(sim_ecc(), [make()], K)
    print("%s: %r" % (case, rep))
    assert rep.fail is None, rep
    if case == "lambda":
        assert rep.last[0][2] == (3, E.FAILED_LAMBDA)


def test_every_iteration_three_sequences_in_one_call():
    rep = run_iterate(sim_ecc(), [converging(), rolling(), lambda_failure()], 6)
    print(rep)
    assert rep.fail is None, rep


# ---------------------------------------------------------------------------------------------- injected bugs
ECC = "b2t_ecc.cu"
BUGS = {
    # name: (patches, where the harness must first fail: "warp" or the iteration of the converging case)
    "hessian_not_f32": ([(ECC, "Hm[0][0] = f32(S[15]); Hm[0][1] = Hm[1][0] = f32(S[16]);", "Hm[0][0] = S[15]; Hm[0][1] = Hm[1][0] = S[16];")], 1),
    "image_mean_not_rounded": ([(ECC, "const double imf = f32(im), tmf = f32(tm);", "const double imf = im, tmf = f32(tm);")], 2),
    "sjt_over_all_pixels": ([(ECC, "for (int k = 0; k < 3; ++k) { acc[9 + k] += J[k]; acc[12 + k] += J[k] * t; }",
                              "for (int k = 0; k < 3; ++k) acc[9 + k] += J[k];"),
                             (ECC, "            if (r.mask) {\n                const double t = (double)T[i];",
                              "            { const double t = (double)T[i]; for (int k = 0; k < 3; ++k) acc[12 + k] += J[k] * t; }\n"
                              "            if (r.mask) {\n                const double t = (double)T[i];")], 2),
    "bilinear_round_15": ([(ECC, "const int X = (X0 + 16 + ad) >> 5", "const int X = (X0 + 15 + ad) >> 5")], "warp"),
    "asin_dropped": ([(ECC, "asin((double)M.m10)", "((double)M.m10)")], 2),
}


def variant(name):
    return L.declare(C.CDLL(build_sim.build_variant("ecc_" + name, BUGS[name][0], units=(ECC, "b2t_nms.cu"))), names=SYMBOLS)


@pytest.mark.parametrize("bug", sorted(BUGS))
def test_injected_bug_fails_where_it_was_made(bug):
    lib = variant(bug)
    where = BUGS[bug][1]
    bad_warp = warp_failures(lib)
    rep = run_iterate(lib, [converging()], 3)
    print(bug, bad_warp[:3], rep)
    if where == "warp":
        assert bad_warp, "the warp stage did not notice"
        assert rep.fail is not None
    else:
        assert not bad_warp
        assert rep.fail is not None and rep.fail[0] == where, rep
