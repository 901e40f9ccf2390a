"""-m gpu: the ECC camera-motion kernels (csrc/b2t_ecc.cu) stage by stage on an H100: the warp stage (``b2t_ecc_warp``) bit for bit
against the cv2 fixtures and the edge maps, the preparation at ds 1 - 5, every iteration of the 8-CTA cluster kernel from its own
previous map within ``ecc_step_ref``'s bound (the distributed-shared-memory combine is what this checks), and one call of mixed
outcomes against single-sequence calls, the oracle and the reference's goldens."""
import ctypes as C
import os
import sys

import numpy as np
import pytest

pytestmark = pytest.mark.gpu
torch = pytest.importorskip("torch")

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "golden"))
import ecc_stages as ES  # noqa: E402
from b200track import _lib as L  # noqa: E402
from b200track import gmc as G  # noqa: E402
from b200track.gmc import EccEstimator  # noqa: E402
from b200track.synth import moved_frame, textured_frame  # noqa: E402
from make_golden_ecc import CASES, frames, warp_plane  # noqa: E402
from oracle import ecc as E  # noqa: E402

GOLD = np.load(os.path.join(HERE, "golden", "ecc.npz"))


def _dev(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def gpu_warp(P, M):
    lib = L.load()
    h, w = P.shape
    Pd = _dev(P)
    out = [torch.zeros((h, w), dtype=torch.float32, device="cuda") for _ in range(3)] + [torch.zeros((h, w), dtype=torch.uint8, device="cuda")]
    Mh = np.ascontiguousarray(np.asarray(M, np.float32).reshape(6))
    G._check(lib, lib.b2t_ecc_warp(Pd.data_ptr(), h, w, Mh.ctypes.data_as(C.POINTER(C.c_float)), *[o.data_ptr() for o in out],
                                   torch.cuda.current_stream().cuda_stream))
    torch.cuda.synchronize()
    return [o.cpu().numpy() for o in out]


def test_warp_stage_bit_exact_with_cv2_fixtures():
    P = np.ascontiguousarray(warp_plane())
    for j in range(len(GOLD["warp_maps"])):
        exp = (GOLD["warp_img"][j], GOLD["warp_gx"][j], GOLD["warp_gy"][j], GOLD["warp_mask"][j])
        assert ES.warp_mismatches(gpu_warp, P, GOLD["warp_maps"][j], exp) == [], j


@pytest.mark.parametrize("shape", ES.EDGE_SHAPES)
def test_warp_stage_edge_maps_bit_exact(shape):
    P = ES.edge_plane(*shape)
    for name, M in ES.EDGE_MAPS:
        assert ES.warp_mismatches(gpu_warp, P, M) == [], (shape, name)


@pytest.mark.parametrize("ds", [1, 2, 3, 4, 5])
def test_prepare_every_downscale(ds):
    for h, w in ((8 * ds, 8 * ds), (8 * ds + 1, 8 * ds + ds - 1 if ds > 1 else 9), (1080, 1920), (1081, 1919)):
        rng = np.random.default_rng(ds * 1000 + h * 7 + w)
        fa, fb = (rng.integers(0, 256, (h, w, 3), dtype=np.uint8) for _ in range(2))
        est = EccEstimator(1, h, w, downscale=ds, max_iter=1)
        est.estimate(_dev(fa[None]))
        est.estimate(_dev(fb[None]))
        assert np.array_equal(est.plane(0, "template"), E.prepare(fa, ds)), (ds, h, w)
        assert np.array_equal(est.plane(0, "current"), E.prepare(fb, ds)), (ds, h, w)


# ---------------------------------------------------------------------------------------------- every iteration
def rotation_shift(s=0):
    base = textured_frame(22 + s, 360, 640, n_rect=300)
    return base, moved_frame(base, 0.3 - 0.1 * s, -1 + 0.5 * s, 1 - 0.25 * s)


def roll(s=0):
    base = textured_frame(7 + s, 120, 160, n_rect=60)
    return base, np.ascontiguousarray(np.roll(base, (2 + s % 2, -3 + s // 2), (0, 1)))


def lambda_failure(s=0):
    if s == 0:
        return tuple(frames(CASES[5]))
    return textured_frame(15 + s, 120, 160, n_rect=50), textured_frame(1015 + s, 120, 160, n_rect=50)


ITER_CASES = {"rotation_shift": (rotation_shift, 12), "roll": (roll, 30), "lambda": (lambda_failure, 6)}


def run_iterate(pairs, K):
    h, w = pairs[0][0].shape[:2]
    est = EccEstimator(len(pairs), h, w)
    f0, f1 = _dev(np.stack([p[0] for p in pairs])), _dev(np.stack([p[1] for p in pairs]))

    def run(k):
        est.reset()
        est.max_iter = k
        est.estimate(f0)
        warps, stat = est.estimate(f1)
        return warps.cpu().numpy(), stat.cpu().numpy()
    planes = [ES.ecc_planes(a, b) for a, b in pairs]
    return ES.iterate(run, planes, K, cluster=8, device=True)


@pytest.mark.parametrize("n_seq", [1, 8])
@pytest.mark.parametrize("case", sorted(ITER_CASES))
def test_every_iteration_from_its_own_previous_map(case, n_seq):
    make, K = ITER_CASES[case]
    rep = run_iterate([make(s) for s in range(n_seq)], K)
    print("%s x %d: %r" % (case, n_seq, rep))
    assert rep.fail is None, rep
    if case == "lambda":
        assert rep.last[0][2] == (GOLD["it5"][1], E.FAILED_LAMBDA)
    if case == "roll":
        assert rep.last[0][2] is None                                    # still iterating after 30: the roll oscillates


def test_mixed_outcomes_in_one_call():
    """Converge, iteration cap, lambda failure and a flat frame in one 8-sequence call: each sequence bitwise its single-sequence
    call, flags and iteration counts those of the oracle, and the reference's on the golden cases (3: flat, 5: lambda)."""
    base = textured_frame(7, 120, 160, n_rect=60)
    pairs = [(base, moved_frame(base, 0.3, 1, -1)), roll(0), tuple(frames(CASES[5])), tuple(frames(CASES[3])),
             (base, moved_frame(base, -0.2, 0.5, 0.5)), roll(1), tuple(frames(CASES[3])), (base, base)]
    golden = {2: 5, 3: 3, 6: 3}
    big = EccEstimator(8, 120, 160)
    big.estimate(_dev(np.stack([p[0] for p in pairs])))
    wb, sb = big.estimate(_dev(np.stack([p[1] for p in pairs])))
    wb, sb = wb.cpu().numpy(), sb.cpu().numpy()
    for s, (f0, f1) in enumerate(pairs):
        one = EccEstimator(1, 120, 160)
        one.estimate(_dev(f0[None]))
        w1, s1 = one.estimate(_dev(f1[None]))
        assert np.array_equal(w1.cpu().numpy()[0], wb[s]) and np.array_equal(s1.cpu().numpy()[0], sb[s]), s
        _, it, fl, _ = E.ecc(E.prepare(f0), E.prepare(f1))
        assert (sb[s, 0], sb[s, 5]) == (it, fl), (s, sb[s, :8], it, fl)
        if s in golden:
            k = golden[s]
            assert (sb[s, 0], sb[s, 5]) == (GOLD["it%d" % k][1], GOLD["fl%d" % k][1]), s
    assert {int(f) for f in sb[:, 5]} == {E.CONVERGED, E.ITER_CAP, E.FAILED_LAMBDA}
