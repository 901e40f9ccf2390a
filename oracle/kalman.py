"""Oracle: constant-velocity Kalman filters of the reference, restated on plain arrays.

TEST INFRASTRUCTURE (see oracle/__init__.py).  Follows tracker/kalman_filter.py:
  * ``KalmanFilter``        (xyah, 'default')   :158-363
  * ``BoTSORTKalmanFilter`` (xywh, 'botsort')   :414-605
  * ``NSAKalmanFilter``     ('strongsort', R scaled by (1-conf)) :607-646
Pinned against those classes executed from /root/reference in the build
container (tests/golden/kalman_*.npz, written by tests/golden/make_golden.py).

dtype notes that matter for bit-level agreement (NumPy 2.x / NEP 50, SURVEY q12):
the reference creates ``mean`` as float32 (from ``STrack._tlwh``) and it only
becomes float64 after the first predict / update / gmc.  While it is float32,
``python_float * mean[3]`` stays float32, so the noise std is rounded to
float32 before it is squared.  ``mean_f32`` flags reproduce that.
"""
import numpy as np
import scipy.linalg

FMT_XYAH, FMT_XYWH, FMT_NSA = 0, 1, 2
FMT_BY_NAME = {"default": FMT_XYAH, "botsort": FMT_XYWH, "strongsort": FMT_NSA}

W_POS = 1.0 / 20
W_VEL = 1.0 / 160

F = np.eye(8)
for _i in range(4):
    F[_i, 4 + _i] = 1.0
H = np.eye(4, 8)


def initiate(fmt, z):
    """kalman_filter.py:190-221 / :435-466.  ``z`` float32[4] -> (mean float32[8], cov)."""
    z = np.asarray(z, dtype=np.float32)
    mean = np.r_[z, np.zeros_like(z)]
    f32 = np.float32
    if fmt == FMT_XYWH:
        # every std entry is np.float32 -> np.square works in float32, cov is float32
        s = [f32(2 * W_POS) * z[2], f32(2 * W_POS) * z[3], f32(2 * W_POS) * z[2], f32(2 * W_POS) * z[3],
             f32(10 * W_VEL) * z[2], f32(10 * W_VEL) * z[3], f32(10 * W_VEL) * z[2], f32(10 * W_VEL) * z[3]]
        cov = np.diag(np.square(np.array(s, dtype=np.float32)))
    else:
        # list mixes np.float32 and Python floats -> float64 array of float32-rounded stds
        s = [f32(2 * W_POS) * z[3], f32(2 * W_POS) * z[3], 1e-2, f32(2 * W_POS) * z[3],
             f32(10 * W_VEL) * z[3], f32(10 * W_VEL) * z[3], 1e-5, f32(10 * W_VEL) * z[3]]
        cov = np.diag(np.square(np.array([float(v) for v in s], dtype=np.float64)))
    return mean, cov


def _q_diag(fmt, mean, f32path):
    """Process noise diagonal, (N,8).  kalman_filter.py:308-318 / :550-560."""
    if f32path:
        m = mean.astype(np.float32)
        wp, wv = np.float32(W_POS), np.float32(W_VEL)
        one = np.ones_like(m[:, 3])
        c2, c5 = np.float32(1e-2) * one, np.float32(1e-5) * one
    else:
        m = mean.astype(np.float64)
        wp, wv = W_POS, W_VEL
        one = np.ones_like(m[:, 3])
        c2, c5 = 1e-2 * one, 1e-5 * one
    if fmt == FMT_XYWH:
        std = [wp * m[:, 2], wp * m[:, 3], wp * m[:, 2], wp * m[:, 3],
               wv * m[:, 2], wv * m[:, 3], wv * m[:, 2], wv * m[:, 3]]
    else:
        std = [wp * m[:, 3], wp * m[:, 3], c2, wp * m[:, 3],
               wv * m[:, 3], wv * m[:, 3], c5, wv * m[:, 3]]
    return np.square(np.stack(std, axis=0)).T  # float32 or float64


def multi_predict(fmt, mean, cov, all_f32=False):
    """kalman_filter.py:289-329 / :534-571.  mean (N,8), cov (N,8,8) -> float64 outputs.

    ``all_f32``: every mean in the batch is still float32 (np.asarray keeps float32), so the
    process noise is evaluated in float32 before being added to the float64 covariance.
    """
    mean = np.asarray(mean)
    cov = np.asarray(cov, dtype=np.float64)
    q = _q_diag(fmt, mean, all_f32)
    mean64 = mean.astype(np.float64)
    new_mean = np.dot(mean64, F.T)
    left = np.dot(F, cov).transpose((1, 0, 2))
    new_cov = np.dot(left, F.T)
    idx = np.arange(8)
    new_cov[:, idx, idx] += q.astype(np.float64)
    return new_mean, new_cov


def project(fmt, mean, cov, mean_f32=False, confidence=0.0):
    """kalman_filter.py:260-287 / :505-532 / :617-631 -> (z_hat float64[4], S float64[4,4])."""
    cov = np.asarray(cov, dtype=np.float64)
    if mean_f32:
        m = np.asarray(mean, dtype=np.float32)
        wp = np.float32(W_POS)
    else:
        m = np.asarray(mean, dtype=np.float64)
        wp = W_POS
    if fmt == FMT_XYWH:
        std = np.array([wp * m[2], wp * m[3], wp * m[2], wp * m[3]])  # float32 stays float32
        r = np.square(std).astype(np.float64)
    else:
        std = [wp * m[3], wp * m[3], 1e-1, wp * m[3]]
        if fmt == FMT_NSA:
            std = [(1 - confidence) * x for x in std]
        if all(isinstance(v, np.float32) for v in std):
            # NSA, float32 mean, float32 confidence: every term is float32 (1e-1 too, via (1 - conf) * 1e-1), so
            # np.square runs in float32 (kalman_filter.py:624-626)
            r = np.square(np.array(std, dtype=np.float32)).astype(np.float64)
        else:
            r = np.square(np.array([float(v) for v in std], dtype=np.float64))
    z_hat = np.dot(H, np.asarray(mean, dtype=np.float64))
    s = np.linalg.multi_dot((H, cov, H.T)) + np.diag(r)
    return z_hat, s


def update(fmt, mean, cov, z, mean_f32=False, confidence=0.0):
    """kalman_filter.py:331-363 / :573-605 / :633-646 -> (mean float64[8], cov float64[8,8])."""
    cov = np.asarray(cov, dtype=np.float64)
    z_hat, s = project(fmt, mean, cov, mean_f32, confidence)
    chol, lower = scipy.linalg.cho_factor(s, lower=True, check_finite=False)
    gain = scipy.linalg.cho_solve((chol, lower), np.dot(cov, H.T).T, check_finite=False).T
    innovation = np.asarray(z, dtype=np.float64) - z_hat
    new_mean = np.asarray(mean, dtype=np.float64) + np.dot(innovation, gain.T)
    new_cov = cov - np.linalg.multi_dot((gain, s, gain.T))
    return new_mean, new_cov


def gating_distance(fmt, mean, cov, measurements, only_position=False, metric="maha", mean_f32=False):
    """kalman_filter.py:365-411.  ``mean_f32``: the mean is still float32, so project rounds the noise std to float32."""
    z_hat, s = project(fmt, mean, cov, mean_f32)
    measurements = np.asarray(measurements, dtype=np.float64)
    if only_position:
        z_hat, s = z_hat[:2], s[:2, :2]
        measurements = measurements[:, :2]
    d = measurements - z_hat
    if metric == "gaussian":
        return np.sum(d * d, axis=1)
    chol = np.linalg.cholesky(s)
    zz = scipy.linalg.solve_triangular(chol, d.T, lower=True, check_finite=False)
    return np.sum(zz * zz, axis=0)


def gmc_apply(mean, cov, warp):
    """tracker/botsort.py:250-269 (multi_gmc) on arrays: mean (N,8), cov (N,8,8), warp (2,3)."""
    mean = np.asarray(mean, dtype=np.float64).copy()
    cov = np.asarray(cov, dtype=np.float64).copy()
    warp = np.asarray(warp, dtype=np.float64)
    r8 = np.kron(np.eye(4, dtype=float), warp[:2, :2])
    t = warp[:2, 2]
    for i in range(mean.shape[0]):
        m = r8.dot(mean[i])
        m[:2] += t
        mean[i] = m
        cov[i] = r8.dot(cov[i]).dot(r8.transpose())
    return mean, cov


# ---- box <-> measurement conversions (tracker/basetrack.py:111-181, float32 arithmetic) ----
def tlbr_to_tlwh_f32(tlbr):
    r = np.asarray(tlbr, dtype=np.float32).copy()
    r[..., 2] -= r[..., 0]
    r[..., 3] -= r[..., 1]
    return r


def tlwh_to_meas_f32(fmt, tlwh):
    """tlwh2xyah (basetrack.py:122-129) or tlwh2xywh with floor division (:144-150)."""
    r = np.asarray(tlwh, dtype=np.float32).copy()
    if fmt == FMT_XYWH:
        r[:2] += r[2:] // 2
    else:
        r[:2] += r[2:] / 2
        r[2] /= r[3]
    return r


def mean_to_tlwh(fmt, mean4):
    """STrack.tlwh, basetrack.py:183-211, in the dtype of ``mean4``."""
    r = np.array(mean4[:4], copy=True)
    if fmt != FMT_XYWH:
        r[2] *= r[3]
    r[:2] -= r[2:] / 2
    return r
