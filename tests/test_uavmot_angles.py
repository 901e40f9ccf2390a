"""not-gpu: the angle certificate of the UAVMOT structure vectors (SURVEY q22).  Detection centres are integers (q9, and tl + wh // 2
of integer boxes), so every offset between two detections of a 1280 x 1280 frame is an integer vector (dx, dy) with |dx|, |dy| <= 1280.
For every such vector off the axes and diagonals, math.atan2(dy, dx) * 180 / math.pi stays further from an integer than the device's
atan2 can move it: the CUDA Math API bounds double atan2 by 2 ulp, the host's by 1 ulp, and the multiply and divide by 180 / pi add one
rounding each -- together under 8 ulp of a value below 180, about 2.6e-13.  On the axes and diagonals the step returns the host's exact
integers (uav_direction), checked here against math.atan2."""
import math

import numpy as np

ULP_180 = np.spacing(180.0)


def test_every_integer_direction_clears_the_device_error():
    r = np.arange(-1280, 1281, dtype=np.float64)
    worst = 1.0
    for dy in r:
        dx = r
        a = np.arctan2(np.full_like(dx, dy), dx) * 180 / math.pi
        off = (dx != 0) & (dy != 0) & (np.abs(dx) != abs(dy))
        g = np.abs(a[off] - np.round(a[off]))
        if len(g):
            worst = min(worst, float(g.min()))
    assert worst > 8 * ULP_180, "an integer direction lies within %.3g of an integer degree" % worst
    assert worst > 1e-9


def test_axes_and_diagonals_are_exact_on_the_host():
    for s in (1.0, 3.0, 397.0, 1280.0):
        for (dx, dy), want in (((s, 0), 0), ((s, s), 45), ((0, s), 90), ((-s, s), 135), ((-s, 0), 180), ((-s, -s), -135),
                               ((0, -s), -90), ((s, -s), -45)):
            assert math.atan2(dy, dx) * 180 / math.pi == want
