"""CPU: the packing part of the gallery kernel's error bound (csrc/b2t_gallery.cu).  The fp16 split of b2t_gallery_pack, restated in
NumPy, must recover the exact dot product of unit vectors within the bound's packing term, on adversarial rows: mixed magnitudes that
put lo (and hi) in the fp16 subnormal range, large norms, dominant elements, identical and opposite rows.  The GPU tests hold the
kernel itself to the whole bound."""
import math
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import gallery_ref as GR                                      # noqa: E402


def _pack_term(d):
    return 3 * 2.0 ** -22 + 2 * 2.0 ** -33 * math.sqrt(d) + 2.0 ** -50


@pytest.mark.parametrize("d", [32, 100, 512, 2048])
def test_split_recovers_the_dot_within_the_packing_term(d):
    rng = np.random.default_rng(d)
    a = GR.adversarial_rows(rng, 120, d)
    b = np.concatenate([GR.adversarial_rows(rng, 60, d), a[:10], -a[10:20]])      # identical (exactly 0) and opposite (exactly 2) rows
    got = GR.packed_dot(GR.pack(a), GR.pack(b))
    ua, ub = GR.unit(a), GR.unit(b)
    err = np.abs(got - ua @ ub.T).max()
    assert err <= _pack_term(d), (err, _pack_term(d))
    assert np.abs(1.0 - got[np.arange(10), 60 + np.arange(10)]).max() <= _pack_term(d)
    assert np.abs(-1.0 - got[10 + np.arange(10), 70 + np.arange(10)]).max() <= _pack_term(d)


def test_adversarial_rows_reach_the_subnormal_range():
    hi, lo = GR.pack(GR.adversarial_rows(np.random.default_rng(0), 200, 512))
    tiny = np.finfo(np.float16).tiny
    assert ((lo != 0) & (np.abs(lo) < tiny)).sum() > 1000        # lo subnormal
    assert ((hi != 0) & (np.abs(hi) < tiny)).sum() > 100         # hi subnormal
    assert np.isfinite(hi.astype(np.float64)).all() and np.abs(hi.astype(np.float64)).max() <= GR.SCALE


def test_bound_values():
    # the figures quoted in the kernel's comment and the header
    assert 2.6e-5 < GR.bound(512) < 2.8e-5
    assert 2.8e-5 < GR.bound(2048) < 3.0e-5
    assert GR.bound(32) < GR.bound(512) < GR.bound(2048) < 1e-4


def test_exact_edges():
    rng = np.random.default_rng(1)
    g = rng.standard_normal((3, 4, 8)).astype(np.float32)
    f = rng.standard_normal((5, 8)).astype(np.float32)
    out = GR.exact(g, [0, 1, 9], f)
    assert np.isinf(out[0]).all()
    np.testing.assert_allclose(out[1], (1 - GR.unit(g[1, :1]) @ GR.unit(f).T)[0], rtol=0, atol=1e-15)
    np.testing.assert_allclose(out[2], (1 - GR.unit(g[2]) @ GR.unit(f).T).min(0), rtol=0, atol=1e-15)
