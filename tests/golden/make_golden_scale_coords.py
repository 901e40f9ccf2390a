"""Writes tests/golden/scale_coords.npz: what the UNMODIFIED reference's ``scale_coords`` (utils/general.py:319-340) returns, with the
``.round()`` of tracker/track.py:240, for canvas boxes mapped back to the source frame at the letterbox geometries a tracker meets:
1080p -> 768 x 1280 (gain 2/3), 720p -> 384 x 640 (1/2), 360 x 640 -> 384 x 640 (gain 1, pad 12), 721 x 1283 -> 768 x 1280
(gain 0.997662, pad 24.3429 -- not the letterbox's 24.5), 480 x 640 -> 960 x 1280 (gain 2) and the identity.  The rows are the
half-integer rows of tests/nms_ref.py plus random boxes, some past the canvas.  Run on the CPU in float32 (the tensor type the
NMS output has) and in float64.  Build container only (needs /root/reference).

    python tests/golden/make_golden_scale_coords.py
"""
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
sys.path.insert(0, os.path.dirname(HERE))
from oracle import refshim  # noqa: E402
import nms_ref as R  # noqa: E402


def rows_for(canvas_hw, src_hw, seed):
    rng = np.random.default_rng(seed)
    half = R.half_integer_rows(canvas_hw, src_hw)
    n = 64
    H, W = canvas_hw
    x1 = rng.uniform(-40, W, n); y1 = rng.uniform(-40, H, n)
    rnd = np.stack([x1, y1, x1 + rng.uniform(0, 300, n), y1 + rng.uniform(0, 300, n), rng.uniform(0, 1, n), rng.integers(0, 80, n)], 1)
    return np.concatenate([half, rnd.astype(np.float32)]).astype(np.float32)


if __name__ == "__main__":
    G = refshim.load_general()
    out = {"src": np.array([s for s, _ in R.GEOMETRIES], np.int64), "canvas": np.array([c for _, c in R.GEOMETRIES], np.int64)}
    for k, (src, canvas) in enumerate(R.GEOMETRIES):
        rows = rows_for(canvas, src, k)
        out["rows%d" % k] = rows
        for name, dt in (("out%d", torch.float32), ("out64_%d", torch.float64)):
            t = torch.from_numpy(rows.copy()).to(dt)                                               # scale_coords works in place
            t[:, :4] = G.scale_coords(canvas, t[:, :4], src, ratio_pad=None).round()          # tracker/track.py:240
            out[name % k] = t.numpy()
    np.savez_compressed(os.path.join(HERE, "scale_coords.npz"), **out)
    print("wrote", os.path.join(HERE, "scale_coords.npz"), [out["rows%d" % k].shape for k in range(len(R.GEOMETRIES))])
