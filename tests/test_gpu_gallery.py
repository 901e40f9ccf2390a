"""gpu: the gallery appearance cost on the tensor cores (b2t_gallery_pack / b2t_gallery_distance, DeepSORT's
matching.nearest_embedding_distance).
  * adversarial rows (mixed magnitudes down to the fp16 subnormal range, large norms, dominant elements, identical and opposite rows)
    against float64 on the exactly normalised rows, within the derived bound (tests/gallery_ref.py), at feature dimensions 32, 100,
    512 and 2048; and against the reference's float32-normalised rows within the bound plus their own normalisation error;
  * the edges: 0 slots, 0 detections, galleries of 1, 99, 100 entries and a 100-entry ring after 101 appends, counts of 0 (+inf) and
    above the budget (clamped), 1024 slots x 1000 detection rows, a budget above one 128-row tile;
  * malformed arguments are refused;
  * the drop-in matching.nearest_embedding_distance on track objects."""
import ctypes as C
import os
import sys

import numpy as np
import pytest

pytestmark = pytest.mark.gpu
torch = pytest.importorskip("torch")

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from b200track import _lib as L                                # noqa: E402
import gallery_ref as GR                                       # noqa: E402


def _ops():
    from b200track.engine import ops
    return ops()


def _device(gal, counts, dets):
    ops = _ops()
    d = gal.shape[-1]
    g = ops.gallery_pack(torch.as_tensor(gal).cuda())
    f = ops.gallery_pack(torch.as_tensor(dets).cuda())
    out = ops.gallery_distance(g, torch.as_tensor(np.asarray(counts, dtype=np.int32)).cuda(), f, d)
    return out.cpu().numpy()


def _exact(gal, counts, dets, normalise=None):
    """float64 reference on the GPU (a checker: torch float64 GEMM, error ~ feat_dim 2^-53)"""
    normalise = normalise or (lambda x: torch.nn.functional.normalize(torch.as_tensor(x, dtype=torch.float64).cuda(), dim=-1))
    t, b, d = gal.shape
    ug = normalise(gal.reshape(t * b, d)).reshape(t, b, d)
    uf = normalise(dets)
    cos = torch.einsum("tbd,md->tbm", ug, uf)
    cnt = torch.as_tensor(np.clip(np.asarray(counts), 0, b)).cuda()
    valid = torch.arange(b, device="cuda")[None, :, None] < cnt[:, None, None]
    return torch.where(valid, 1.0 - cos, torch.full_like(cos, np.inf)).min(1).values.cpu().numpy()


def _check(gal, counts, dets):
    got = _device(gal, counts, dets)
    exp = _exact(gal, counts, dets)
    assert got.shape == exp.shape
    fin = np.isfinite(exp)
    assert (np.isinf(got) == ~fin).all()
    err = np.abs(got[fin] - exp[fin]).max() if fin.any() else 0.0
    assert err <= GR.bound(gal.shape[-1]), (err, GR.bound(gal.shape[-1]))
    return got, exp


@pytest.mark.parametrize("d", [32, 100, 512, 2048])
def test_adversarial_within_bound(d):
    rng = np.random.default_rng(100 + d)
    t, b, m = 40, 100, 300
    gal = GR.adversarial_rows(rng, t * b, d).reshape(t, b, d)
    dets = GR.adversarial_rows(rng, m, d)
    dets[:20] = gal[np.arange(20), rng.integers(0, 50, size=20)]       # identical rows: distance exactly 0
    dets[20:40] = -gal[20 + np.arange(20), 0]                           # opposite rows: distance exactly 2 to one-entry galleries
    counts = rng.integers(1, b + 1, size=t)
    counts[:20] = 50
    counts[20:40] = 1
    got, exp = _check(gal, counts, dets)
    assert np.abs(got[np.arange(20), np.arange(20)]).max() <= GR.bound(d)
    assert np.abs(got[20 + np.arange(20), 20 + np.arange(20)] - 2.0).max() <= GR.bound(d)
    # against the reference's own float32-normalised rows (cal_cosine_distance): the bound plus their normalisation error, bounded per
    # pair by Cauchy-Schwarz from |r^ - u| of the two rows.  The reference's float32 norm overflows on the 1e30 rows, so those are
    # scaled down first (the device result does not depend on a row's scale beyond the bound).
    def tame(x):
        return np.where(np.abs(x).max(-1, keepdims=True) > 1e15, x * np.float32(1e-25), x).astype(np.float32)
    gal, dets = tame(gal), tame(dets)
    got = _device(gal, counts, dets)
    ref = _exact(gal, counts, dets, normalise=lambda x: torch.as_tensor(GR.reference_normalised(x), dtype=torch.float64).cuda())
    rg = np.linalg.norm(GR.reference_normalised(gal.reshape(-1, d)).astype(np.float64) - GR.unit(gal.reshape(-1, d)), axis=1).max()
    rf = np.linalg.norm(GR.reference_normalised(dets).astype(np.float64) - GR.unit(dets), axis=1).max()
    assert rg < 1e-5 and rf < 1e-5
    assert np.abs(got - ref).max() <= GR.bound(d) + rg * (1 + rf) + rf


def test_gallery_sizes_and_ring():
    rng = np.random.default_rng(7)
    d, b = 512, 100
    feats = rng.standard_normal((101, d)).astype(np.float32)
    ring = np.zeros((b, d), dtype=np.float32)
    for i, f in enumerate(feats):                                         # 101 appends into a ring of 100: entry 0 is overwritten
        ring[i % b] = f
    gal = np.zeros((5, b, d), dtype=np.float32)
    counts = [1, 99, 100, 100, 0]
    gal[0, :1] = feats[:1]
    gal[1, :99] = feats[:99]
    gal[2] = feats[:100]
    gal[3] = ring
    dets = np.concatenate([feats[:1] * 3, feats[100:], rng.standard_normal((30, d)).astype(np.float32)])
    got, _ = _check(gal, counts, dets)
    assert np.isinf(got[4]).all()
    assert abs(got[3, 1]) <= GR.bound(d) and got[2, 1] > 0.5                          # entry 100 is in the ring, not in the first 100
    assert abs(got[2, 0]) <= GR.bound(d) and got[3, 0] > 0.5                          # entry 0 was overwritten


def test_counts_clamped_and_long_gallery():
    rng = np.random.default_rng(8)
    gal = rng.standard_normal((3, 300, 64)).astype(np.float32)            # a budget of three 128-row tiles
    dets = np.concatenate([gal[0, 257:259], gal[1, 5:6], rng.standard_normal((7, 64)).astype(np.float32)])
    got, _ = _check(gal, [300, 1000, -4], dets)
    assert np.isinf(got[2]).all() and abs(got[0, 0]) <= GR.bound(64)


def test_empty_inputs():
    ops = _ops()
    g = ops.gallery_pack(torch.zeros((0, 100, 512), device="cuda"))
    f = ops.gallery_pack(torch.ones((7, 512), device="cuda"))
    assert ops.gallery_distance(g, torch.zeros(0, dtype=torch.int32, device="cuda"), f, 512).shape == (0, 7)
    g = ops.gallery_pack(torch.ones((3, 100, 512), device="cuda"))
    f = ops.gallery_pack(torch.zeros((0, 512), device="cuda"))
    assert ops.gallery_distance(g, torch.ones(3, dtype=torch.int32, device="cuda"), f, 512).shape == (3, 0)


def test_cap_slots_dmax_rows():
    rng = np.random.default_rng(9)
    t, b, d, m = 1024, 100, 512, 1000
    gal = rng.standard_normal((t, b, d)).astype(np.float32)
    dets = rng.standard_normal((m, d)).astype(np.float32)
    dets[:200] += 3 * gal[rng.integers(0, t, size=200), rng.integers(0, b, size=200)]     # some small distances
    _check(gal, rng.integers(1, b + 1, size=t), dets)


def test_refusals():
    lib = L.load()
    ops = _ops()
    g = ops.gallery_pack(torch.ones((2, 4, 64), device="cuda"))
    f = ops.gallery_pack(torch.ones((3, 64), device="cuda"))
    cnt = torch.ones(2, dtype=torch.int32, device="cuda")
    out = torch.empty((2, 3), dtype=torch.float64, device="cuda")
    p = lambda t: C.c_void_p(t.data_ptr())                                        # noqa: E731
    assert lib.b2t_gallery_distance(p(g), p(cnt), 2, 0, p(f), 3, 64, p(out), None) == L.EINVAL          # budget 0
    assert lib.b2t_gallery_distance(p(g), p(cnt), 2, 4, p(f), 3, 0, p(out), None) == L.EINVAL           # feat_dim 0
    assert lib.b2t_gallery_distance(C.c_void_p(g.data_ptr() + 2), p(cnt), 2, 4, p(f), 3, 64, p(out), None) == L.EINVAL
    assert b"aligned" in lib.b2t_last_error()
    assert lib.b2t_gallery_distance(None, p(cnt), 2, 4, p(f), 3, 64, p(out), None) == L.EINVAL
    assert lib.b2t_gallery_pack(None, 2, 64, p(g), None) == L.EINVAL
    assert lib.b2t_gallery_row_halves(64) == 128 and lib.b2t_gallery_row_halves(65) == 256 and lib.b2t_gallery_row_halves(0) == 0
    # the Python wrapper refuses what the kernel would read out of bounds
    with pytest.raises(L.B2TError):
        ops.gallery_distance(g.float(), cnt, f, 64)                                   # not packed fp16
    with pytest.raises(L.B2TError):
        ops.gallery_distance(g, cnt, f, 128)                                          # packed for another feat_dim
    with pytest.raises(L.B2TError):
        ops.gallery_distance(g, cnt.long(), f, 64)                                    # counts not int32
    with pytest.raises(L.B2TError):
        ops.gallery_distance(g, cnt[:1], f, 64)                                       # one count per slot
    with pytest.raises(L.B2TError):
        ops.gallery_distance(g[:, ::2], cnt, f, 64)                                   # not contiguous
    with pytest.raises(L.B2TError):
        ops.gallery_pack(torch.ones((3, 64), device="cuda", dtype=torch.float64))


def test_zero_rows_give_nan_as_the_reference():
    """a zero feature row normalises to NaN in the reference (0 / 0) and ndarray.min propagates it; so does the kernel"""
    rng = np.random.default_rng(12)
    gal = rng.standard_normal((3, 100, 128)).astype(np.float32)
    gal[1, 40] = 0                                                                    # inside the gallery: slot 1 is NaN throughout
    gal[2, 90] = 0                                                                    # beyond slot 2's count: not read
    dets = rng.standard_normal((5, 128)).astype(np.float32)
    dets[3] = 0                                                                       # a zero detection row: NaN column
    got = _device(gal, [100, 100, 60], dets)
    assert np.isnan(got[1]).all() and np.isnan(got[:, 3]).all()
    keep = np.array([0, 1, 2, 4])
    exp = _exact(gal, [100, 100, 60], dets)
    assert np.isfinite(got[0][keep]).all() and np.isfinite(got[2][keep]).all()
    assert np.abs(got[[0, 2]][:, keep] - exp[[0, 2]][:, keep]).max() <= GR.bound(128)


class _Track:
    def __init__(self, feats):
        self.features = list(feats)


def test_dropin_nearest_embedding_distance():
    tdir = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "yolov7-tracker_b200", "tracker")
    sys.path.insert(0, tdir)
    try:
        import matching
    finally:
        sys.path.remove(tdir)
    rng = np.random.default_rng(11)
    d = 512
    tracks = [_Track(rng.standard_normal((n, d)).astype(np.float32)) for n in (1, 7, 100, 42)]
    dets = [_Track(rng.standard_normal((1, d)).astype(np.float32)) for _ in range(9)]
    dets[3].features = [tracks[2].features[17] * 2]
    got = matching.nearest_embedding_distance(tracks, dets)
    exp = np.stack([(1 - GR.unit(np.asarray(t.features)) @ GR.unit(np.asarray([x.features[-1] for x in dets])).T).min(0) for t in tracks])
    assert got.shape == (4, 9) and got.dtype == np.float64
    assert np.abs(got - exp).max() <= GR.bound(d)
    assert abs(got[2, 3]) <= GR.bound(d)
    assert matching.nearest_embedding_distance([], dets).shape == (0, 9)
    assert matching.nearest_embedding_distance(tracks, []).shape == (4, 0)


def test_dropin_matches_the_per_track_path_on_extractor_like_rows():
    """On rows like the ReID extractor's (non-negative after its ReLU and average pool, large cosines), the one-launch drop-in agrees
    with float64 to the 5e-6 the per-track split-fp16 path it replaces is held to (tests/test_gpu_parity.py), and with that path
    itself; the derived bound is a worst case, not the error seen at the 0.15 gate."""
    tdir = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "yolov7-tracker_b200", "tracker")
    sys.path.insert(0, tdir)
    try:
        import matching
    finally:
        sys.path.remove(tdir)
    rng = np.random.default_rng(13)
    d = 512
    ident = np.abs(rng.standard_normal((30, d)))
    def feat(i):
        return np.maximum(ident[i] + 0.55 * rng.standard_normal(d), 0).astype(np.float32)
    tracks = [_Track([feat(i) for _ in range(int(rng.integers(1, 101)))]) for i in range(30)]
    dets = [_Track([feat(int(i))]) for i in rng.integers(0, 30, size=60)]
    got = matching.nearest_embedding_distance(tracks, dets)
    det_f = np.asarray([x.features[-1] for x in dets])
    exp = np.stack([(1 - GR.unit(np.asarray(t.features)) @ GR.unit(det_f).T).min(0) for t in tracks])
    old = np.stack([(1. - matching.cal_cosine_distance(np.asarray(t.features), det_f)).min(axis=0) for t in tracks])
    assert ((exp > 0.1) & (exp < 0.2)).sum() > 20                                     # pairs near the 0.15 gate
    assert np.abs(got - exp).max() < 5e-6
    assert np.abs(got - old).max() < 1e-5
