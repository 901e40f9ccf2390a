"""gpu: the assignment solver's cases (tests/lap_cases.py) at full size on the nvcc build -- the only tier where the 16 warps of
a CTA solve their components truly concurrently -- and the drop-in matching.linear_assignment on the large-weight
counterexamples.  Each case prints the counters it reached, the certified gap and, in float32, the largest objective
shortfall over its bound."""
import ctypes as C
import os
import sys

import numpy as np
import pytest

import lap_cases as LC
import lap_ref as R
from b200track import _lib as L

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu
PKG = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "yolov7-tracker_b200")


class GpuBackend:
    def __init__(self):
        self.lib = L.load()

    def dev(self, a):
        return torch.from_numpy(np.ascontiguousarray(a)).cuda()

    def ptr(self, t):
        return C.c_void_p(t.data_ptr())

    def host(self, t):
        return t.cpu().numpy()

    def sync(self):
        torch.cuda.synchronize()


@pytest.fixture(scope="module")
def be():
    assert torch.cuda.is_available()
    return GpuBackend()


def test_version(be):
    assert be.lib.b2t_version() == 107


@pytest.mark.parametrize("dtype", [L.F64, L.F32], ids=["f64", "f32"])
@pytest.mark.parametrize("case", sorted(LC.CASES))
def test_lap_case(be, case, dtype):
    rep = LC.CASES[case](be, dtype, True)
    print("%s[%s]: %s" % (case, "f64" if dtype == L.F64 else "f32", rep.line()))


def test_dropin_linear_assignment_large_weights(be):
    """tracker/matching.linear_assignment (imported by its bare name, as track.py does) on the counterexamples to the old rule:
    the reference's matches and unmatched lists."""
    saved = {k: sys.modules.pop(k) for k in ("matching", "kalman_filter") if k in sys.modules}
    sys.path.insert(0, os.path.join(PKG, "tracker"))
    try:
        import matching
        for name, (cost, t, xopt, _) in LC._regression_problems().items():
            m, ua, ub = matching.linear_assignment(cost, t)
            _, x = R.solve(cost, t)
            rows = np.nonzero(x >= 0)[0]
            assert [list(p) for p in np.asarray(m).reshape(-1, 2)] == [[int(i), int(x[i])] for i in rows], name
            assert list(ua) == list(np.nonzero(x < 0)[0]), name
            assert list(ub) == list(np.nonzero(R.y_of(x, cost.shape[1]) < 0)[0]), name
    finally:
        sys.path.remove(os.path.join(PKG, "tracker"))
        for k in ("matching", "kalman_filter"):
            sys.modules.pop(k, None)
        sys.modules.update(saved)
