"""not-gpu: pins for the ECC stage harnesses (tests/ecc_stages.py, tests/ecc_step_ref.py).  oracle/ecc.py's warp against
cv2.warpAffine on the edge maps and planes the GPU tier checks the kernel with (cv2 may be missing on a GPU machine, so the pin is
made here), and the oracle's own NumPy iteration inside ``ecc_step_ref``'s reachable set at both cluster sizes."""
import numpy as np
import pytest

import ecc_stages as ES
import ecc_step_ref as R
from b200track.synth import moved_frame, textured_frame
from oracle import ecc as E

cv2 = pytest.importorskip("cv2")


@pytest.mark.parametrize("shape", ES.EDGE_SHAPES + [(31, 47)])
def test_edge_maps_oracle_equals_cv2_warpaffine(shape):
    P = ES.edge_plane(*shape)
    h, w = shape
    Pf = P.astype(np.float32)
    gx = cv2.filter2D(Pf, -1, np.array([[-0.5, 0, 0.5]], np.float32))
    gy = cv2.filter2D(Pf, -1, np.array([[-0.5], [0], [0.5]], np.float32))
    flags = cv2.INTER_LINEAR + cv2.WARP_INVERSE_MAP
    for name, M in ES.EDGE_MAPS:
        exp = (cv2.warpAffine(Pf, M, (w, h), flags=flags), cv2.warpAffine(gx, M, (w, h), flags=flags),
               cv2.warpAffine(gy, M, (w, h), flags=flags),
               cv2.warpAffine(np.ones_like(P), M, (w, h), flags=cv2.INTER_NEAREST + cv2.WARP_INVERSE_MAP))
        got = ES.warp_expected(P, M)
        for k, a, b in zip(("img", "gx", "gy", "mask"), got, exp):
            assert np.array_equal(a, b), (shape, name, k)


def test_edge_maps_hit_their_edges():
    """The tie maps put rint(. * 1024) on .5 and the edge maps move the mask's border, so the harness tests what it claims."""
    P = ES.edge_plane(31, 47)
    maps = dict(ES.EDGE_MAPS)
    assert (maps["tie_x"][0, 2] * 1024) % 1 == 0.5 and (maps["tie_col"][1, 0] * 3 * 1024) % 1 == 0.5
    assert E.warp_nearest_mask(31, 47, maps["near_lo"]).all()
    assert not E.warp_nearest_mask(31, 47, maps["near_lo_out"])[0].any()
    assert E.warp_nearest_mask(31, 47, maps["near_hi"]).all()
    assert not E.warp_nearest_mask(31, 47, maps["near_hi_out"])[-1].any()
    X, Y = E._coords(maps["tap_m1"], 31, 47, False)
    assert (X >> 5).min() == -1 and (Y >> 5).min() == -1
    X, Y = E._coords(maps["tap_end"], 31, 47, False)
    assert (X >> 5).max() + 1 == 47 and (Y >> 5).max() + 1 == 31
    assert ES.warp_expected(P, maps["tap_m1"])[0][0, 0] != 0


@pytest.mark.parametrize("cluster", [1, 8])
def test_oracle_iteration_inside_its_own_set(cluster):
    """oracle/ecc.py's step on its NumPy (pairwise) sums lands in the set ``step_set`` derives from the correctly rounded sums,
    every iteration of a converging rotation + shift at 180 x 320 working pixels."""
    base = textured_frame(22, 360, 640, n_rect=300)
    t, im = E.prepare(base), E.prepare(moved_frame(base, 0.3, -1, 1))
    gx, gy = E.gradients(im)
    M, last, forks = np.eye(2, 3, dtype=np.float32), -1.0, 0
    for k in range(1, 20):
        st = R.step_set(t, im, M, last, cluster=cluster)
        M2, rho, fl = E.step(E.sums(t, im, gx, gy, M), M)
        flag = fl or (E.CONVERGED if abs(rho - last) < 1e-5 else R.CONTINUE)
        assert st.contains(M2, flag, rho), (k, M2, flag, rho, st.outcomes, st.rho_lo, st.rho_hi)
        forks += st.forks
        if flag:
            break
        M, last = M2, rho
    assert flag == E.CONVERGED and k > 2
    print("cluster %d: %d iterations, %d forks" % (cluster, k, forks))


def test_bound_too_loose_is_a_failure():
    """A sum bound that covers several float32 values of the Hessian raises instead of passing."""
    base = textured_frame(22, 120, 160, n_rect=60)
    t, im = E.prepare(base), E.prepare(moved_frame(base, 0.3, -1, 1))
    S, Rb = R.sums_with_bound(t, im, np.eye(2, 3, dtype=np.float32), 8)
    with pytest.raises(R.BoundTooLoose):
        R.step_from_sums(S, [abs(s) * 1e-5 for s in S], np.eye(2, 3, dtype=np.float32), -1.0)
    assert R.step_from_sums(S, Rb, np.eye(2, 3, dtype=np.float32), -1.0).forks == 0
