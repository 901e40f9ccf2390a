"""-m gpu: the ECC camera-motion estimator (csrc/b2t_ecc.cu, one thread-block cluster per sequence) on an H100 through the C ABI:
against the UNMODIFIED reference's results (tests/golden/ecc.npz) and oracle/ecc.py, bitwise reproducibility across calls and across
the number of sequences per call, reset(), and the drop-in ``botsort.GMC(method='ecc')`` / ``multi_gmc``."""
import os
import sys
import types

import numpy as np
import pytest

pytestmark = pytest.mark.gpu
torch = pytest.importorskip("torch")

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "golden"))
from b200track import _lib as L  # noqa: E402
from b200track.gmc import EccEstimator, ecc_rho  # noqa: E402
from b200track.synth import textured_frame  # noqa: E402
from make_golden_ecc import CASES, frames, plane_digest  # noqa: E402
from oracle import ecc as E  # noqa: E402
from oracle import gmc as OG  # noqa: E402
from oracle import kalman as OK  # noqa: E402

GOLD = np.load(os.path.join(HERE, "golden", "ecc.npz"))


def _dev(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


@pytest.mark.parametrize("k", range(len(CASES)))
def test_vs_reference_golden(k):
    """Same flags and iteration counts as the reference's findTransformECC, every warp within 0.01 px at the corners of the half-scale
    frame, and the prepared template bit for bit."""
    case = CASES[k]
    est = EccEstimator(1, case["h"], case["w"])
    hh, ww = case["h"] // 2, case["w"] // 2
    worst = 0.0
    for i, f in enumerate(frames(case)):
        warps, stat = est.estimate(_dev(f[None]))
        H, st = warps[0].cpu().numpy(), stat[0].cpu().numpy()
        assert st[5] == GOLD["fl%d" % k][i] and st[0] == GOLD["it%d" % k][i], (k, i, st[:8], GOLD["fl%d" % k][i], GOLD["it%d" % k][i])
        d = OG.corner_displacement(H, GOLD["H%d" % k][i].astype(np.float64), hh, ww)
        worst = max(worst, d)
        assert d < 0.01, (k, i, H, GOLD["H%d" % k][i])
        if i == 0:
            assert np.array_equal(plane_digest(est.plane(0, "template")), GOLD["plane_sha%d" % k][0])
    print("case %d: worst corner displacement vs the reference %.2e px" % (k, worst))


def test_batch_of_eight_equals_single_calls_and_repeats_bitwise():
    h, w = 720, 1280
    base = [textured_frame(200 + s, h, w, n_rect=600) for s in range(8)]
    seqs = [[b, np.ascontiguousarray(np.roll(b, (s % 3 + 1, -(s % 4) - 1), (0, 1)))] for s, b in enumerate(base)]
    big = EccEstimator(8, h, w)
    for i in range(2):
        wb, sb = big.estimate(_dev(np.stack([seqs[s][i] for s in range(8)])))
    wb, sb = wb.clone(), sb.clone()
    for s in range(8):
        one = EccEstimator(1, h, w)
        for i in range(2):
            w1, s1 = one.estimate(_dev(seqs[s][i][None]))
        assert torch.equal(w1[0], wb[s]) and torch.equal(s1[0], sb[s]), s
    big.reset()
    for i in range(2):
        w2, s2 = big.estimate(_dev(np.stack([seqs[s][i] for s in range(8)])))
    assert torch.equal(w2, wb) and torch.equal(s2, sb)
    assert (sb[:, 5].cpu().numpy() == L.ECC_CONVERGED).all() and (sb[:, 0].cpu().numpy() > 1).all()


def test_vs_oracle_and_reset_starts_new_template():
    h, w = 360, 640
    a = textured_frame(301, h, w, n_rect=300)
    b = textured_frame(302, h, w, n_rect=300)
    est = EccEstimator(1, h, w)
    orc = E.EccOracle()
    for f in (a, np.roll(a, (2, -3), (0, 1)), np.roll(a, (4, -1), (0, 1))):
        warps, stat = est.estimate(_dev(f[None]))
        H, it, fl, rho = orc.apply(np.ascontiguousarray(f))
        st = stat[0].cpu().numpy()
        assert st[0] == it and st[5] == fl
        np.testing.assert_allclose(warps[0].cpu().numpy(), H, rtol=0, atol=1e-5)
        if it:
            assert abs(ecc_rho(stat.cpu().numpy())[0] - rho) < 1e-6
    est.reset()
    warps, stat = est.estimate(_dev(b[None]))
    assert stat[0, 5].item() == L.ECC_FIRST_FRAME and np.array_equal(est.plane(0, "template"), E.prepare(b))
    warps, stat = est.estimate(_dev(np.roll(b, (0, 2), (0, 1))[None]))
    assert stat[0, 7].item() == 1 and abs(warps[0, 0, 2].item() - 1.0) < 0.05            # a 2-px roll = 1 half-scale px


def test_dropin_gmc_ecc_and_multi_gmc(capsys):
    sys.path.insert(0, os.path.join(os.path.dirname(HERE), "yolov7-tracker_b200", "tracker"))
    import botsort as B
    with pytest.raises(NotImplementedError):
        B.GMC(method='sift')
    h, w = 240, 320
    base = textured_frame(77, h, w, n_rect=120)
    seq = [base, np.ascontiguousarray(np.roll(base, (2, -4), (0, 1))), np.full_like(base, 90)]
    gmc = B.GMC(method='ecc', downscale=2)
    est = EccEstimator(1, h, w)
    for i, f in enumerate(seq):
        H = gmc.apply(f if i != 1 else _dev(f), None)
        we, _ = est.estimate(_dev(f[None]))
        assert isinstance(H, np.ndarray) and H.dtype == np.float32 and H.shape == (2, 3)
        assert np.array_equal(H, we[0].cpu().numpy().astype(np.float32))
        out = capsys.readouterr().out
        if i == 0:
            assert np.array_equal(H, np.eye(2, 3, dtype=np.float32)) and "find transform failed" not in out
        elif i == 1:
            Hmove = H
            assert abs(H[0, 2] + 2.0) < 0.05 and abs(H[1, 2] - 1.0) < 0.05 and "find transform failed" not in out
        else:
            assert np.array_equal(H, np.eye(2, 3, dtype=np.float32)) and "Warning: find transform failed. Set warp as identity" in out
    rng = np.random.default_rng(5)
    mean = rng.normal(0, 50, (7, 8)) + np.array([300, 200, 40, 80, 0, 0, 0, 0])
    A = rng.normal(0, 1, (7, 8, 8))
    cov = A @ A.transpose(0, 2, 1) + np.eye(8)
    tracks = [types.SimpleNamespace(mean=mean[i].copy(), cov=cov[i].copy()) for i in range(7)]
    B.multi_gmc(tracks, Hmove)
    em, ec = OK.gmc_apply(mean, cov, Hmove)
    np.testing.assert_allclose(np.stack([t.mean for t in tracks]), em, rtol=0, atol=1e-9)
    np.testing.assert_allclose(np.stack([t.cov for t in tracks]), ec, rtol=0, atol=1e-9)
