"""Writes tests/golden/kalman_gating.npz by running the UNMODIFIED reference's KalmanFilter.gating_distance
(tracker/kalman_filter.py:365-411), for KalmanFilter and NSAKalmanFilter, read through B2T_REFERENCE_ROOT like the other
generators (oracle/refshim.py).  Run in the build container only: ``python tests/golden/make_golden_gating.py``.

Per filter: 12 states -- 4 fresh from initiate (float32 mean, the reference's own dtype before the first predict), the same 4 after
one predict (float64), and those predicted means cast back to float32 -- at the edges of tests/kalman_bounds.py (centres up to 8192,
heights 1 - 4000 px, aspect ratios 0.02 - 50), each against 24 measurements (near, far, and at the other states), for both metrics and
both only_position values.  The float32-mean states pin where project rounds the noise std to float32 (SURVEY q12)."""
import os
import sys

import numpy as np
import scipy

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, os.path.join(ROOT, "yolov7-tracker_b200"))

from oracle import refshim  # noqa: E402
import kalman_bounds as KB  # noqa: E402

VERS = dict(numpy=np.__version__, scipy=scipy.__version__)


def fixture(kf, fmt, seed):
    rng = np.random.default_rng(seed)
    z = KB.measurements(rng, 4, fmt)
    z[0, 3] = np.float32(1.5)                                       # a 1.5 px box
    m0, c0 = zip(*[kf.initiate(zi) for zi in z])
    mp, cp = kf.multi_predict(np.stack(m0), np.stack(c0))
    means = list(m0) + list(mp) + [m.astype(np.float32) for m in mp]
    covs = [np.asarray(c, np.float64) for c in c0] + list(cp) + list(cp)
    meas = np.concatenate([KB.near(rng, np.stack([m.astype(np.float64) for m in means]), fmt, 2.0), z,
                           KB.measurements(rng, 8, fmt)]).astype(np.float32)[:24]
    out = dict(mean=np.stack([m.astype(np.float64) for m in means]), mean_f32=np.array([m.dtype == np.float32 for m in means]),
               cov=np.stack(covs), meas=meas)
    for op in (False, True):
        for metric in ("maha", "gaussian"):
            out["gate_%d_%s" % (op, metric)] = np.stack([kf.gating_distance(m, c, meas.astype(np.float64), op, metric)
                                                         for m, c in zip(means, covs)])
    return out


def main():
    ref = refshim.load()
    out = {}
    for name, cls, fmt, seed in (("default", ref.kalman_filter.KalmanFilter, 0, 31), ("strongsort", ref.kalman_filter.NSAKalmanFilter, 2, 32)):
        for k, v in fixture(cls(), fmt, seed).items():
            out["%s_%s" % (name, k)] = v
    np.savez_compressed(os.path.join(HERE, "kalman_gating.npz"), **out, **{"ver_" + k: v for k, v in VERS.items()})
    print("kalman_gating ok")


if __name__ == "__main__":
    main()
