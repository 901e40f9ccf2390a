"""Drop-in for the reference's ``tracker/kalman_filter.py`` -- same classes, same NumPy-in /
NumPy-out methods, arithmetic on the GPU (csrc/b2t_kalman.cuh through libb200track.so).

  KalmanFilter         xyah   reference :158-411
  BoTSORTKalmanFilter  xywh   reference :414-605
  NSAKalmanFilter      xyah + confidence-scaled R   reference :607-646
  NaiveKalmanFilter    7-d xyar, reference :23-155 -- NOT accelerated: the reference's own
                       multi_predict for it raises on NumPy >= 1.24 (SURVEY q11), so the format is dead.

These per-call wrappers exist for API fidelity (third-party trackers that drive the filter
object by object).  The fast path -- ByteTrack / BoT-SORT / SORT ``update`` -- never calls them:
it runs the whole frame in one kernel (b200track.engine.TrackEngine).
There is no CPU fallback: without a CUDA device these methods raise.
"""
import numpy as np

import _b2t_path  # noqa: F401
from b200track import _lib as L
from b200track import engine as _eng

# 0.95 quantile of the chi-square distribution with N degrees of freedom (reference :11-20)
chi2inv95 = {1: 3.8415, 2: 5.9915, 3: 7.8147, 4: 9.4877, 5: 11.070, 6: 12.592, 7: 14.067, 8: 15.507, 9: 16.919}

import torch  # noqa: E402


def _flags_for(mean):
    return L.FLAG_MEAN_F32 if np.asarray(mean).dtype == np.float32 else 0


class _GpuKalman(object):
    _fmt = L.FMT_XYAH
    ndim = 4

    def __init__(self):
        self._std_weight_position = 1. / 20
        self._std_weight_velocity = 1. / 160
        self._motion_mat = np.eye(8)
        for i in range(4):
            self._motion_mat[i, 4 + i] = 1.
        self._update_mat = np.eye(4, 8)

    # -- helpers
    @staticmethod
    def _ops():
        return _eng.ops()

    def initiate(self, measurement):
        ops = self._ops()
        z = ops.dev(np.asarray(measurement, dtype=np.float64).reshape(1, 4), torch.float64)
        mean, cov = ops.kalman_initiate(L.F64, self._fmt, z)
        mean = mean[0].cpu().numpy().astype(np.float32)            # reference: float32 mean (from STrack._tlwh)
        cov = cov[0].cpu().numpy()
        if self._fmt == L.FMT_XYWH:
            cov = cov.astype(np.float32)                           # reference: float32 covariance for botsort
        return mean, cov

    def predict(self, mean, covariance):
        m, c = self.multi_predict(np.asarray(mean)[None], np.asarray(covariance)[None])
        return m[0], c[0]

    def multi_predict(self, mean, covariance):
        ops = self._ops()
        mean = np.asarray(mean)
        q_f32 = mean.dtype == np.float32
        m = ops.dev(mean.astype(np.float64), torch.float64)
        c = ops.dev(np.asarray(covariance, dtype=np.float64), torch.float64)
        ops.kalman_predict(L.F64, self._fmt, m, c, None, q_f32)
        return m.cpu().numpy(), c.cpu().numpy()

    def project(self, mean, covariance, confidence=None):
        ops = self._ops()
        m = ops.dev(np.asarray(mean, dtype=np.float64).reshape(1, 8), torch.float64)
        c = ops.dev(np.asarray(covariance, dtype=np.float64).reshape(1, 8, 8), torch.float64)
        fl = ops.dev(np.array([_flags_for(mean)], dtype=np.int32), torch.int32)
        cf = None if confidence is None else ops.dev(np.array([confidence], dtype=np.float32), torch.float32)
        pm, ps = ops.kalman_project(L.F64, self._fmt, m, c, fl, cf)
        return pm[0].cpu().numpy(), ps[0].cpu().numpy()

    def update(self, mean, covariance, measurement, confidence=None):
        ops = self._ops()
        m = ops.dev(np.asarray(mean, dtype=np.float64).reshape(1, 8), torch.float64)
        c = ops.dev(np.asarray(covariance, dtype=np.float64).reshape(1, 8, 8), torch.float64)
        z = ops.dev(np.asarray(measurement, dtype=np.float64).reshape(1, 4), torch.float64)
        fl = ops.dev(np.array([_flags_for(mean)], dtype=np.int32), torch.int32)
        cf = None if confidence is None else ops.dev(np.array([confidence], dtype=np.float32), torch.float32)
        ops.kalman_update(L.F64, self._fmt, m, c, z, None, cf, fl)
        return m[0].cpu().numpy(), c[0].cpu().numpy()

    def gating_distance(self, mean, covariance, measurements, only_position=False, metric='maha'):
        if metric not in ('maha', 'gaussian'):
            raise ValueError('invalid distance metric')
        ops = self._ops()
        m = ops.dev(np.asarray(mean, dtype=np.float64).reshape(8), torch.float64)
        c = ops.dev(np.asarray(covariance, dtype=np.float64).reshape(8, 8), torch.float64)
        z = ops.dev(np.asarray(measurements, dtype=np.float64).reshape(-1, 4), torch.float64)
        return ops.kalman_gating(L.F64, self._fmt, m, c, z, only_position, 0 if metric == 'maha' else 1,
                                 _flags_for(mean) != 0).cpu().numpy()


class KalmanFilter(_GpuKalman):
    """8-d (x, y, a, h, vx, vy, va, vh) constant-velocity filter."""
    _fmt = L.FMT_XYAH

    def project(self, mean, covariance):
        return _GpuKalman.project(self, mean, covariance)

    def update(self, mean, covariance, measurement):
        return _GpuKalman.update(self, mean, covariance, measurement)


class BoTSORTKalmanFilter(_GpuKalman):
    """8-d (x, y, w, h, vx, vy, vw, vh) filter of BoT-SORT."""
    _fmt = L.FMT_XYWH

    def project(self, mean, covariance):
        return _GpuKalman.project(self, mean, covariance)

    def update(self, mean, covariance, measurement):
        return _GpuKalman.update(self, mean, covariance, measurement)


class NSAKalmanFilter(KalmanFilter):
    """StrongSORT's NSA filter: measurement noise scaled by (1 - confidence)."""
    _fmt = L.FMT_NSA

    def project(self, mean, covariance, confidence=.0):
        return _GpuKalman.project(self, mean, covariance, confidence)

    def update(self, mean, covariance, measurement, confidence=.0):
        # the reference default `.0` is a Python float: no float32 rounding of (1 - conf) then
        conf = None if (isinstance(confidence, float) and confidence == 0.0) else confidence
        return _GpuKalman.update(self, mean, covariance, measurement, conf)


class NaiveKalmanFilter(object):
    """7-d (x, y, area, ratio) SORT filter.  Present for import compatibility only."""

    def __init__(self):
        pass

    def _dead(self, *a, **k):
        raise NotImplementedError("kalman_format='naive' is not accelerated: the reference's own NaiveKalmanFilter."
                                  "multi_predict raises ValueError on NumPy >= 1.24 (ragged array), so the format is unusable "
                                  "there too.  Use 'default', 'botsort' or 'strongsort'.")

    initiate = predict = multi_predict = project = update = _dead
