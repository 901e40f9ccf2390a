"""Build container only: runs the UNMODIFIED reference ECC estimator (tracker/botsort.py ``GMC(method='ecc', downscale=2)``, host
OpenCV) over seeded sequences and stores what it returns in tests/golden/ecc.npz.  The frames are rebuilt from the seeds by the tests
without OpenCV (b200track.synth.textured_frame + integer rolls / synth.moved_frame).

Per case and frame: ``H{k}`` the returned 2 x 3 float32 matrix, ``it{k}`` the iterations findTransformECC ran (found by re-running it on
the reference's own planes with an iteration cap of 1 ... 100 until the result stops changing; for a failure, the first cap that
raises), ``fl{k}`` the flags (include/b200track.h B2T_ECC_*; the failure kind from the exception's message).  Per-stage fixtures: the
planes cv2 prepares (cvtColor + GaussianBlur + resize) of every frame as SHA-256 digests ``plane_sha{k}`` (``plane_digest``), and in full
(``plane{k}``) for the two small cases, and ``warp_*``: cv2.warpAffine of a small seeded plane
(and of its filter2D gradients, and of an all-ones mask) under seeded Euclidean maps."""
import contextlib
import io
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
for p in (ROOT, os.path.join(ROOT, "yolov7-tracker_b200")):
    sys.path.insert(0, p)
from b200track.synth import moved_frame, textured_frame  # noqa: E402

FIRST_FRAME, CONVERGED, ITER_CAP, FAILED_NAN, FAILED_LAMBDA = 1, 2, 4, 8, 16

# kind "roll": integer rolls (dy, dx) of one textured frame; "move": synth.moved_frame(angle, tx, ty); "flat": a textured frame, then a
# flat one (rho is NaN in the first iteration); "other": a textured frame, then an unrelated one (lambda_d <= 0 after two updates).
# The oracle follows the reference to < 1e-6 on the converging cases; the iteration-cap and failure cases wander (see test_oracle_ecc).
CASES = [
    dict(kind="roll", seed=11, h=720, w=1280, n_rect=600, moves=[(0, 0), (1, -1), (2, -3), (4, -5), (6, -8), (9, -11)]),
    dict(kind="roll", seed=12, h=481, w=643, n_rect=300, moves=[(0, 0), (1, -1), (2, -3), (-3, 4), (5, 5), (6, -8)]),
    dict(kind="move", seed=22, h=360, w=640, n_rect=300, moves=[(0, 0, 0), (0.1, 0.5, 0.5), (0.3, -1, 1), (0.25, 2, 0), (-0.15, 1, -2)]),
    dict(kind="flat", seed=40, h=120, w=160, n_rect=50, moves=[None, None]),
    dict(kind="move", seed=13, h=360, w=640, n_rect=300, moves=[(0, 0, 0), (-0.5, -2, 1.5)]),
    dict(kind="other", seed=15, h=120, w=160, n_rect=50, moves=[None, None]),
]


def frames(case):
    base = textured_frame(case["seed"], case["h"], case["w"], n_rect=case["n_rect"])
    if case["kind"] == "roll":
        return [np.ascontiguousarray(np.roll(base, m, (0, 1))) for m in case["moves"]]
    if case["kind"] == "move":
        return [base if m == (0, 0, 0) else moved_frame(base, *m) for m in case["moves"]]
    if case["kind"] == "flat":
        return [base, np.full_like(base, 90)]
    return [base, textured_frame(case["seed"] + 1000, case["h"], case["w"], n_rect=case["n_rect"])]


WARP_MAPS = [(0.0, 0.37, -1.21), (0.003, 1.37, -2.2), (-0.02, -3.5, 4.25), (0.05, 0.0, 0.0)]


SMALL = (3, 5)                       # cases whose planes are stored in full (60 x 80); the others as digests only


def plane_digest(plane):
    """SHA-256 of a prepared uint8 plane's bytes, with its shape: (32,) uint8."""
    import hashlib
    a = np.ascontiguousarray(plane, np.uint8)
    h = hashlib.sha256(np.array(a.shape, np.int64).tobytes())
    h.update(a.tobytes())
    return np.frombuffer(h.digest(), np.uint8).copy()


def warp_map(theta, tx, ty):
    c, s = np.float32(np.cos(theta)), np.float32(np.sin(theta))
    return np.array([[c, -s, tx], [s, c, ty]], np.float32)


def warp_plane(seed=5, h=31, w=47):
    return np.random.default_rng(seed).integers(0, 256, (h, w), dtype=np.uint8)


if __name__ == "__main__":
    import cv2
    from oracle import refshim
    crit = lambda k: (cv2.TERM_CRITERIA_EPS | cv2.TERM_CRITERIA_COUNT, k, 1e-5)      # noqa: E731

    def run(t, im, k):
        H = np.eye(2, 3, dtype=np.float32)
        try:
            cv2.findTransformECC(t, im, H, cv2.MOTION_EUCLIDEAN, crit(k), None, 1)
            return H, None
        except cv2.error as e:
            return H, str(e)

    def iterations(t, im):
        Hf, ef = run(t, im, 100)
        lo, hi = 1, 100
        while lo < hi:
            m = (lo + hi) // 2
            H, e = run(t, im, m)
            if (e is not None) if ef else np.array_equal(H, Hf):
                hi = m
            else:
                lo = m + 1
        if ef:
            fl = FAILED_NAN if "NaN" in ef else FAILED_LAMBDA
        else:                                          # stopped by eps unless one more iteration still moves the map
            fl = CONVERGED if lo < 100 or np.array_equal(run(t, im, 101)[0], Hf) else ITER_CAP
        return lo, fl

    def cv_prepare(f):
        g = cv2.cvtColor(f, cv2.COLOR_BGR2GRAY)
        g = cv2.GaussianBlur(g, (3, 3), 1.5)
        return cv2.resize(g, (f.shape[1] // 2, f.shape[0] // 2))

    out = {}
    for k, case in enumerate(CASES):
        gmc = refshim.load().botsort.GMC(method='ecc', downscale=2)
        Hs, its, fls, planes, warned = [], [], [], [], []
        for i, f in enumerate(frames(case)):
            buf = io.StringIO()
            with contextlib.redirect_stdout(buf):
                H = gmc.apply(f)
            planes.append(cv_prepare(f))
            Hs.append(np.asarray(H, np.float32))
            warned.append("find transform failed" in buf.getvalue())
            if i == 0:
                its.append(0); fls.append(FIRST_FRAME)
            else:
                it, fl = iterations(gmc.prevFrame, planes[-1])
                its.append(it); fls.append(fl)
                assert warned[-1] == bool(fl & (FAILED_NAN | FAILED_LAMBDA))
        out["H%d" % k] = np.stack(Hs)
        out["it%d" % k] = np.array(its, np.int32)
        out["fl%d" % k] = np.array(fls, np.int32)
        out["plane_sha%d" % k] = np.stack([plane_digest(p) for p in planes])
        if k in SMALL:
            out["plane%d" % k] = np.stack(planes)
        print(k, its, fls, flush=True)
    P = warp_plane()
    Pf = P.astype(np.float32)
    gx = cv2.filter2D(Pf, -1, np.array([[-0.5, 0, 0.5]], np.float32))
    gy = cv2.filter2D(Pf, -1, np.array([[-0.5], [0], [0.5]], np.float32))
    flags = cv2.INTER_LINEAR + cv2.WARP_INVERSE_MAP
    maps = [warp_map(*m) for m in WARP_MAPS]
    size = (P.shape[1], P.shape[0])
    out["warp_maps"] = np.stack(maps)
    out["warp_img"] = np.stack([cv2.warpAffine(Pf, M, size, flags=flags) for M in maps])
    out["warp_gx"] = np.stack([cv2.warpAffine(gx, M, size, flags=flags) for M in maps])
    out["warp_gy"] = np.stack([cv2.warpAffine(gy, M, size, flags=flags) for M in maps])
    out["warp_mask"] = np.stack([cv2.warpAffine(np.ones_like(P), M, size, flags=cv2.INTER_NEAREST + cv2.WARP_INVERSE_MAP) for M in maps])
    np.savez_compressed(os.path.join(ROOT, "tests", "golden", "ecc.npz"), **out)
    print(sorted(out))
