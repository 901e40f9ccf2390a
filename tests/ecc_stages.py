"""TEST INFRASTRUCTURE: the ECC stage harnesses shared by the GPU tier (tests/test_gpu_ecc_stages.py) and the simulator tier
(tests/test_hostsim_ecc_stages.py).  Each takes a runner -- the device build or a simulator build of csrc/b2t_ecc.cu -- and returns
what it found instead of asserting, so that an injected bug can be shown to fail at the stage or iteration it was made in.

  * ``EDGE_MAPS`` / ``edge_planes``: warp maps on the edges of warpAffine's fixed point (ties of rint(x * 1024) at 1/2048 px, taps
    on index -1 / h / w, the nearest mask's + 512 >> 10 edge) and planes from 2 x 2 up to one larger than the warp kernel's grid.
    tests/test_oracle_ecc_edges.py pins oracle/ecc.py against cv2.warpAffine on all of them.
  * ``warp_mismatches``: the warp stage (``b2t_ecc_warp``) bit for bit against the oracle.
  * ``iterate``: every iteration from the kernel's own previous map, against ``ecc_step_ref.step_set``."""
import numpy as np

import ecc_step_ref as R
from oracle import ecc as E

T2048 = 1.0 / 2048


def _m(a00, a01, a02, a10, a11, a12):
    return np.array([[a00, a01, a02], [a10, a11, a12]], np.float32)


# (name, map): warpAffine with WARP_INVERSE_MAP, M maps destination (x, y) to source
EDGE_MAPS = [
    ("tie_x", _m(1, 0, 3 * T2048, 0, 1, 0)),                    # rint(tx * 1024) on .5: round half to even, 1 and 2
    ("tie_xy", _m(1, 0, -5 * T2048, 0, 1, 7 * T2048)),
    ("tie_xy_odd", _m(1, 0, 0.5 + T2048, 0, 1, -(0.25 + 3 * T2048))),
    ("tie_col", _m(1, 0, 0, T2048, 1, 0)),                      # m10 * x * 1024 = x / 2: a tie on every odd column
    ("tie_row", _m(1, T2048, 0, 0, 1, 0)),                      # m01 * y * 1024 = y / 2 on every odd row
    ("tap_m1", _m(1, 0, -1 + 1.0 / 64, 0, 1, -1 + 1.0 / 64)),     # first taps on index -1
    ("tap_end", _m(1, 0, 1.0 / 64, 0, 1, 1.0 / 64)),              # last taps on index h / w
    ("near_lo", _m(1, 0, -0.5, 0, 1, -0.5)),                    # X0 + 512 == 0: mask column / row 0 still inside
    ("near_lo_out", _m(1, 0, -0.5 - 1.0 / 1024, 0, 1, -0.5 - 1.0 / 1024)),
    ("near_hi", _m(1, 0, 0.5 - 1.0 / 1024, 0, 1, 0.5 - 1.0 / 1024)),
    ("near_hi_out", _m(1, 0, 0.5, 0, 1, 0.5)),                  # the last column / row maps to w / h: outside
    ("rot_edge", _m(np.cos(0.02), -np.sin(0.02), -0.5, np.sin(0.02), np.cos(0.02), 0.5 - 1.0 / 1024)),
    ("far", _m(1, 0, -40.0, 0, 1, 13.5)),                      # most taps outside
]

# (h, w): the smallest planes, a tall one, and one larger than the 528 x 256-thread grid (the grid-stride loop wraps)
EDGE_SHAPES = [(2, 2), (8, 8), (8192, 16), (397, 403)]


def edge_plane(h, w, seed=9):
    return np.random.default_rng(seed + h * 31 + w).integers(0, 256, (h, w), dtype=np.uint8)


def warp_expected(P, M):
    """(img, gx, gy, mask) of the warp stage by oracle/ecc.py."""
    gx, gy = E.gradients(P)
    return (E.warp_linear(P.astype(np.float32), M), E.warp_linear(gx, M), E.warp_linear(gy, M),
            E.warp_nearest_mask(P.shape[0], P.shape[1], M))


def warp_mismatches(warp, P, M, expected=None):
    """Names of the warp outputs ``warp(P, M) -> (img, gx, gy, mask)`` gets wrong (bit for bit)."""
    exp = warp_expected(P, M) if expected is None else expected
    got = warp(P, M)
    return [n for n, a, b in zip(("img", "gx", "gy", "mask"), got, exp) if not np.array_equal(np.asarray(a), np.asarray(b))]


class IterReport:
    def __init__(self):
        self.fail = None                 # (iteration, sequence, what) of the first departure
        self.worst_ratio = 0.0           # largest sum bound / |sum| met
        self.worst_rho = 0.0             # largest |device rho - interval centre| / half-width
        self.forks = 0                   # forks summed over the checked iterations
        self.max_forks = 0
        self.checked = 0                 # iterations checked
        self.last = None                 # per sequence: (iterations, flag, map) at the end

    def __repr__(self):
        return ("checked %d iterations, %d forks (at most %d in one), largest rho err / bound %.3f, largest sum bound / |sum| %.2e, "
                "first failure %s" % (self.checked, self.forks, self.max_forks, self.worst_rho, self.worst_ratio, self.fail))


def iterate(run, planes, K, cluster, device, eps=1e-5):
    """Every iteration from the kernel's own previous map.  ``run(k) -> (warps (S, 2, 3), stat (S, 8))`` runs the kernel with
    max_iter = k on the sequences' second frames after a reset and their first; ``planes[s] = (template, current)``.  Iteration k
    of sequence s must be an outcome of ``step_set`` applied to the map and rho run k - 1 reported, with its rho inside the
    interval, until the sequence stops; later runs must then repeat it.  Stops at the first departure (``IterReport.fail``)."""
    S = len(planes)
    rep = IterReport()
    state = [(np.eye(2, 3, dtype=np.float32), -1.0, None)] * S        # (map, rho, stopped at (it, flag) or None)
    cache = {}
    for k in range(1, K + 1):
        warps, stat = run(k)
        warps, stat = np.asarray(warps), np.asarray(stat)
        rhos = np.ascontiguousarray(stat[:, 1:3]).view(np.float64)[:, 0]
        for s in range(S):
            M, last, stopped = state[s]
            Mk = warps[s].astype(np.float32)
            if not np.array_equal(Mk.astype(np.float64), warps[s]):
                rep.fail = (k, s, "map is not float32")
                return rep
            if stopped is not None:
                if (stat[s, 0], stat[s, 5]) != stopped or R.bits(Mk) != R.bits(M):
                    rep.fail = (k, s, "a stopped sequence changed: %s" % (stat[s, :8],))
                    return rep
                continue
            if stat[s, 0] != k or stat[s, 7] != 1:
                rep.fail = (k, s, "stat %s" % (stat[s, :8],))
                return rep
            key = (s, R.bits(M), last)
            if key not in cache:
                cache[key] = R.step_set(planes[s][0], planes[s][1], M, last, eps, cluster, device)
            st = cache[key]
            rep.checked += 1
            rep.forks += st.forks
            rep.max_forks = max(rep.max_forks, st.forks)
            rep.worst_ratio = max(rep.worst_ratio, st.sum_ratio)
            if st.rho_hi > st.rho_lo:
                rep.worst_rho = max(rep.worst_rho, abs(float(rhos[s]) - (st.rho_lo + st.rho_hi) / 2) / ((st.rho_hi - st.rho_lo) / 2))
            fl = int(stat[s, 5])
            ref_fl = R.CONTINUE if fl == E.ITER_CAP else fl
            if not st.contains(Mk, ref_fl, float(rhos[s])):
                rep.fail = (k, s, "map %s flag %d rho %r not among %d outcome(s) %s, rho in [%r, %r]" % (
                    Mk.reshape(6).tolist(), fl, float(rhos[s]), len(st.outcomes), sorted(st.outcomes)[:2], st.rho_lo, st.rho_hi))
                return rep
            state[s] = (Mk, float(rhos[s]), None if fl == E.ITER_CAP else (k, fl))
    rep.last = state
    return rep


def ecc_planes(f0, f1, ds=2):
    return E.prepare(f0, ds), E.prepare(f1, ds)
