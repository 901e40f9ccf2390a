"""-m gpu: every element-wise kernel of the ReID extractor (csrc/b2t_reid.cu) and b2t_image_nhwc16 through the C ABI on an H100, against
float64 references (tests/reid_kernel_ref.py) at the shapes, types and edges where such kernels go wrong: within one 16-bit ulp, exact
where the operation is exact.  Then the extractor as a whole: batch sizes across the capacity buckets against oracle/reid.py, bitwise
reproducibility, and features_from_frame against the crops the reference cuts."""
import ctypes as C
import os
import sys

import numpy as np
import pytest

pytestmark = pytest.mark.gpu
torch = pytest.importorskip("torch")

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import reid_kernel_ref as K  # noqa: E402
from b200track import _lib as L  # noqa: E402

DTS = ["fp16", "bf16"]
WRAP = 132 * 16 * 256                    # grid_for's cap x 256 threads: sizes above this run the grid-stride loops more than once


class TorchMem:
    def put(self, a):
        a = np.ascontiguousarray(a)
        if a.dtype == np.uint16:
            a = a.view(np.int16)
        return torch.from_numpy(a.copy()).cuda()

    def ptr(self, t):
        return C.c_void_p(t.data_ptr())

    def get(self, t):
        torch.cuda.synchronize()
        a = t.cpu().numpy()
        return a.view(np.uint16) if a.dtype == np.int16 else a

    def stream(self):
        return C.c_void_p(torch.cuda.current_stream().cuda_stream)


MEM = TorchMem()


@pytest.fixture(scope="module")
def lib():
    return L.load()


# ---------------------------------------------------------------- b2t_reid_crops

CROP_WINDOWS = [  # (h, w, pitch_px, x0, y0, frame_h, odd_lead)
    (1, 1, 5, 2, 1, 3, 1), (1, 1, 1, 0, 0, 1, 0), (1, 90, 91, 1, 0, 1, 3), (70, 1, 1, 0, 0, 70, 5),                   # 1x1, 1xN, Nx1
    (40, 25, 30, 0, 3, 50, 1), (100, 50, 50, 0, 0, 100, 0),                                                           # upscale, frame corners
    (128, 64, 64, 0, 0, 128, 7), (128, 64, 100, 36, 9, 137, 2),                                                        # exactly 64 x 128
    (256, 128, 128, 0, 0, 256, 0), (256, 128, 140, 12, 4, 260, 1),                                                     # exactly 2x
    (129, 65, 65, 0, 0, 129, 3), (333, 177, 181, 4, 2, 335, 1), (700, 31, 35, 4, 0, 700, 9), (17, 300, 300, 0, 5, 22, 1),
]


@pytest.mark.parametrize("dt", DTS)
def test_reid_crops_within_1ulp_of_float64_and_cv2(lib, dt):
    """Windows of frames (pitch != 3 w, odd byte offsets, windows touching every frame edge) surrounded by sentinel 255 pixels;
    n = 260 crops > one pass of the grid-stride loop."""
    rng = np.random.default_rng(1 if dt == "fp16" else 2)
    base = len(CROP_WINDOWS)
    wins = CROP_WINDOWS + [(int(rng.integers(1, 300)), int(rng.integers(1, 150)), 0, 0, 0, 0, int(rng.integers(0, 4))) for _ in range(260 - base)]
    wins = [w if w[2] else (w[0], w[1], w[1] + w[6], w[6] % 3, w[6] % 2, w[0] + w[6] % 2 + 1, w[6]) for w in wins]
    assert 260 * 128 * 64 > WRAP
    buf, rows, contents = K.crop_frame(rng, wins)
    out = K.run_crops(lib, MEM, buf, rows, len(wins), dt)
    worst, worst_cv = 0.0, 0.0
    for i, win in enumerate(contents):
        worst = max(worst, K.assert_within_1ulp(out[i, :, :, :3], K.crop_ref(win), dt, "crop %d %s" % (i, win.shape), floor=2.0 ** -8))
        worst_cv = max(worst_cv, K.assert_within_1ulp(out[i, :, :, :3], K.crop_cv2(win), dt, "crop %d vs cv2" % i, floor=2.0 ** -8))
    assert (out[:, :, :, 3:] == 0).all()
    print("reid_crops %s: max %.3f ulp vs float64, %.3f ulp vs cv2.resize" % (dt, worst, worst_cv))


# ---------------------------------------------------------------- max pools

POOL3 = [(1, 1, 8), (1, 7, 64), (9, 1, 8), (2, 2, 512), (7, 5, 64), (8, 6, 8), (13, 11, 512), (128, 64, 64)]
POOL2 = [(2, 2, 8), (6, 4, 64), (10, 14, 512), (128, 64, 64)]


@pytest.mark.parametrize("dt", DTS)
@pytest.mark.parametrize("k,h,w,c", [(3,) + s for s in POOL3] + [(2,) + s for s in POOL2])
def test_maxpool_exact_vs_torch(lib, dt, k, h, w, c):
    """All-negative inputs (a padding of 0 instead of -inf shows at every border); n chosen so that the grid-stride loop wraps."""
    ho, wo = ((h + 1) // 2, (w + 1) // 2) if k == 3 else (h // 2, w // 2)
    n = max(2, WRAP // (ho * wo * (c // 8)) + 1)
    rng = np.random.default_rng(k * 1000 + h * 10 + w + c)
    x = K.round16(-np.abs(rng.normal(3, 1, (n, h, w, c))) - 0.01, dt)
    got = K.run_maxpool(lib, MEM, x, k, dt)
    assert np.array_equal(got, K.maxpool_ref(x, dt, k))


# ---------------------------------------------------------------- add + ReLU

@pytest.mark.parametrize("dt", DTS)
@pytest.mark.parametrize("n", [8, 8 * 1001, 8 * (WRAP + 12345)])
def test_add_relu_exact(lib, dt, n):
    rng = np.random.default_rng(n)
    a = K.rand16(rng, n, dt, scale=2.0)
    b = K.rand16(rng, n, dt, scale=2.0)
    q = n // 4
    b[:q] = a[:q] ^ np.uint16(0x8000)                                          # x + (-x): +0
    got = K.run_add_relu(lib, MEM, a, b, dt)
    tdt = torch.float16 if dt == "fp16" else torch.bfloat16
    ta, tb = (torch.from_numpy(v.view(np.int16)).view(tdt) for v in (a, b))
    exp = torch.relu(ta.float() + tb.float()).to(tdt).view(torch.int16).numpy().view(np.uint16)
    assert np.array_equal(got, exp)
    K.assert_within_1ulp(got, K.add_relu_ref(a, b, dt), dt, "add_relu")
    assert (got[:q] == 0).all()


# ---------------------------------------------------------------- BatchNorm with batch statistics

BN_NPIX = [1, 7, 32, 8192, 8192 * 33]
BN_CAP_NPIX = 512 * 8192                 # with c = 16 or 512 this reaches the 1056-block grid cap of the statistics pass


def _bn_case(lib, dt, c, n_pix, ratio, relu, inplace, seed):
    rng = np.random.default_rng(seed)
    x, gamma, beta = K.bn_inputs(rng, n_pix + 5, c, dt, ratio)
    y, _ = K.run_bn(lib, MEM, x, n_pix, c, gamma, beta, dt, relu, inplace)
    mean, var = K.bn_stats_ref(x, dt, n_pix, c)
    worst, rows = 0.0, max(1, (1 << 22) // c)
    for r0 in range(0, n_pix, rows):                                          # the check in slices: 2^26-element cases stay in memory
        r1 = min(n_pix, r0 + rows)
        ref = K.bn_apply_ref(x[r0:r1], dt, mean, var, gamma, beta, 1e-5, relu)
        worst = max(worst, K.assert_within_1ulp(y[r0:r1], ref, dt, "bn c=%d n_pix=%d mean/std=%g relu=%d rows %d.." % (c, n_pix, ratio, relu, r0)))
    tail = x[n_pix:] if inplace else np.full_like(x[n_pix:], 0x7777)
    assert np.array_equal(y[n_pix:], tail), "rows past n_pix written"
    if n_pix == 1:
        assert np.array_equal(y[0], K.round16(np.maximum(beta, 0) if relu else beta, dt))
    return worst


@pytest.mark.parametrize("dt", DTS)
@pytest.mark.parametrize("c", [8, 16, 32, 64, 128, 256, 512])
def test_batchnorm_every_width_and_size(lib, dt, c):
    """Every allowed c at n_pix from 1 up to the grid cap (n_pix * c kept to 2^23 elements, 2^26 for the grid-cap case)."""
    sizes = [min(n, (1 << 23) // c) for n in BN_NPIX] + ([min(BN_CAP_NPIX, (1 << 26) // c)] if c in (16, 512) else [])
    if c in (16, 512):
        assert lib.b2t_batchnorm_workspace_bytes(sizes[-1], c) == (2 * c + 1056 * 2 * c) * 8
    worst = 0.0
    for k, n_pix in enumerate(sizes):
        worst = max(worst, _bn_case(lib, dt, c, n_pix, 0, k % 2, (k // 2) % 2, c * 10 + k))
    print("bn %s c=%d: max %.3f ulp" % (dt, c, worst))


@pytest.mark.parametrize("dt", DTS)
@pytest.mark.parametrize("ratio", [0, 10, 100, 1000])
@pytest.mark.parametrize("relu,inplace", [(0, 0), (1, 1)])
def test_batchnorm_large_mean_over_std(lib, dt, ratio, relu, inplace):
    """mean/std up to 1000: a one-pass E[x^2] - mean^2 from float partials loses the variance here."""
    worst = max(_bn_case(lib, dt, 64, 8192 * 4, ratio, relu, inplace, ratio + 7 * relu + 3 * inplace),
                _bn_case(lib, dt, 512, 8192, ratio, relu, inplace, ratio + 1))
    print("bn %s mean/std=%d: max %.3f ulp" % (dt, ratio, worst))


def test_batchnorm_no_state_through_workspace_and_bitwise_repeatable(lib):
    rng = np.random.default_rng(5)
    x1, g1, b1 = K.bn_inputs(rng, 8192 * 4, 512, "fp16", 10)
    x2, g2, b2 = K.bn_inputs(rng, 8192 * 33, 64, "fp16", 100)
    nb = max(lib.b2t_batchnorm_workspace_bytes(8192 * 4, 512), lib.b2t_batchnorm_workspace_bytes(8192 * 33, 64))
    ws = MEM.put(np.zeros(nb // 8))
    K.run_bn(lib, MEM, x1, 8192 * 4, 512, g1, b1, "fp16", 0, 0, ws=ws)
    y_after, _ = K.run_bn(lib, MEM, x2, 8192 * 33, 64, g2, b2, "fp16", 1, 0, ws=ws)
    fresh, _ = K.run_bn(lib, MEM, x2, 8192 * 33, 64, g2, b2, "fp16", 1, 0)
    assert np.array_equal(y_after, fresh)
    for dt, c, n_pix in (("fp16", 64, 512 * 8192 // 8), ("bf16", 512, 8192 * 33)):
        x, g, b = K.bn_inputs(np.random.default_rng(c), n_pix, c, dt, 100)
        outs = [K.run_bn(lib, MEM, x, n_pix, c, g, b, dt, 1, 0)[0] for _ in range(5)]
        for o in outs[1:]:
            assert np.array_equal(o, outs[0]), "batch-statistics BatchNorm differs between identical calls"


# ---------------------------------------------------------------- average pool + L2 norm

@pytest.mark.parametrize("dt", DTS)
@pytest.mark.parametrize("hw", [1, 32, 33, 1000])
def test_avgpool_l2norm_vs_float64(lib, dt, hw):
    rng = np.random.default_rng(hw)
    n = 6
    x = K.rand16(rng, (n, hw, 512), dt)
    x[1:4] = K.round16(np.abs(K.widen16(x[1:4], dt)), dt)                      # post-ReLU rows, as in the network
    x[5] = 0                                                                  # all-zero row: 0 / 0 = NaN, as x.div(x.norm()) gives
    got = K.run_avgpool(lib, MEM, x, n, hw, dt)
    ref = K.avgpool_ref(x, dt, n, hw)
    assert np.abs(got[:5] - ref[:5]).max() <= 1e-6                            # unit vectors: 1e-6 relative to the norm
    assert np.isnan(got[5]).all()


# ---------------------------------------------------------------- YOLOv7-tiny's input

@pytest.mark.parametrize("dt", DTS)
def test_image_nhwc16_exact(lib, dt):
    g = torch.Generator().manual_seed(3)
    img = (torch.randn((2, 3, 67, 45), generator=g) * 3).cuda()
    tdt = torch.float16 if dt == "fp16" else torch.bfloat16
    out = torch.full((2, 67, 45, 16), 7, dtype=torch.int16, device="cuda")
    rc = lib.b2t_image_nhwc16(C.c_void_p(img.data_ptr()), C.c_void_p(out.data_ptr()), 2, 67, 45, K.CODE[dt], MEM.stream())
    assert rc == 0, lib.b2t_detect_last_error()
    torch.cuda.synchronize()
    o = out.view(tdt)
    assert torch.equal(o[..., :3].view(torch.int16), img.permute(0, 2, 3, 1).to(tdt).view(torch.int16))
    assert (out[..., 3:] == 0).all()


def test_argument_errors(lib):
    """Each entry point's documented limits: B2T_EINVAL and a message, nothing launched."""
    EINVAL = -1
    p = C.c_void_p(256)
    s = MEM.stream()
    assert lib.b2t_maxpool3x3s2(p, p, 1, 4, 4, 12, 1, s) == EINVAL and b"multiple of 8" in lib.b2t_detect_last_error()
    assert lib.b2t_maxpool2x2s2(p, p, 1, 5, 4, 8, 1, s) == EINVAL and b"even" in lib.b2t_detect_last_error()
    assert lib.b2t_maxpool2x2s2(p, p, 1, 4, 3, 8, 1, s) == EINVAL
    assert lib.b2t_add_relu(p, p, p, 12, 1, s) == EINVAL and b"multiple of 8" in lib.b2t_detect_last_error()
    for c in (4, 12, 520):
        assert lib.b2t_batchnorm_batch_stats(p, p, 10, c, p, p, 1e-5, 0, p, 1, s) == EINVAL
        assert lib.b2t_batchnorm_workspace_bytes(10, c) == 0
    assert b"c % 8" in lib.b2t_detect_last_error()
    assert lib.b2t_batchnorm_batch_stats(p, p, 10, 24, p, p, 1e-5, 0, p, 1, s) == EINVAL and b"256" in lib.b2t_detect_last_error()
    assert lib.b2t_batchnorm_workspace_bytes(10, 24) == 0
    assert lib.b2t_batchnorm_batch_stats(p, p, 0, 64, p, p, 1e-5, 0, p, 1, s) == EINVAL
    assert lib.b2t_avgpool_l2norm(p, p, 1, 4, 256, 1, s) == EINVAL and b"512" in lib.b2t_detect_last_error()
    assert lib.b2t_reid_crops(p, p, 1, p, 7, s) == EINVAL
    assert lib.b2t_image_nhwc16(p, p, 1, 0, 4, 1, s) == EINVAL
    torch.cuda.synchronize()


# ---------------------------------------------------------------- the extractor

@pytest.fixture(scope="module")
def extractors():
    from b200track.reid import ReidExtractor
    from oracle import reid as R
    sd = R.seeded_state_dict(3)
    return sd, {m: ReidExtractor(sd, bn_mode=m) for m in ("batch", "running")}


@pytest.mark.parametrize("bn_mode", ["batch", "running"])
@pytest.mark.parametrize("n", [1, 2, 31, 32, 33, 100, 257])
def test_extractor_batch_sizes_vs_oracle(extractors, bn_mode, n):
    """Sizes across the capacity buckets (32, 64, ...): the padding rows repeat crop 0 and must stay out of the statistics."""
    from oracle import reid as R
    sd, ext = extractors
    crops = R.seeded_crops(100 + n, n)
    got = ext[bn_mode](crops)
    with torch.no_grad():
        exp = R.forward(sd, R.preprocess(crops), batch_stats=bn_mode == "batch").numpy()
    cos = (got * exp).sum(1)
    print("reid %s n=%d: min cosine %.6f, max |d| %.2e" % (bn_mode, n, float(cos.min()), float(np.abs(got - exp).max())))
    if n == 1 and bn_mode == "batch":
        # one crop: every last-stage BatchNorm sees 8 x 4 positions; the features are still defined
        assert np.isfinite(got).all()
    assert cos.min() > 0.9999 and np.abs(got - exp).max() < 2e-3


def test_extractor_bitwise_reproducible_across_interleaved_calls(extractors):
    from oracle import reid as R
    _, ext = extractors
    e = ext["batch"]
    sets = {n: R.seeded_crops(500 + n, n) for n in (40, 10, 257)}
    seen = {}
    for n in (40, 10, 40, 257, 40, 10, 257):
        f = e(sets[n])
        if n in seen:
            assert np.array_equal(f, seen[n]), "features of the same %d crops differ between calls" % n
        seen[n] = f


def test_features_from_frame_vs_reference_slicing(extractors):
    """Fractional boxes inside [0, W] x [0, H] (what clip_coords hands over), boxes touching each edge, 1-px-wide boxes: the features of
    ori_img[int(y1):int(y2), int(x1):int(x2)] (botsort.py:291-311) computed by the oracle."""
    from b200track.synth import textured_frame
    from oracle import reid as R
    sd, ext = extractors
    H, W = 360, 500
    frame = textured_frame(11, H, W, n_rect=200)
    rng = np.random.default_rng(4)
    x1 = rng.uniform(0, W - 40, 30); y1 = rng.uniform(0, H - 60, 30)
    boxes = [np.stack([x1, y1, x1 + rng.uniform(2, 40, 30), y1 + rng.uniform(2, 60, 30)], 1),
             np.array([[0.0, 0.0, 30.7, 50.2], [W - 20.5, 0.0, W, 40.0], [0.0, H - 33.3, 25.9, H], [W - 11.0, H - 70.0, W, H],
                       [100.2, 50.0, 101.9, 120.0], [0.0, 10.0, 1.0, H], [5.5, 0.0, W, 1.99], [0.0, 0.0, W, H]])]
    tlbr = np.concatenate(boxes)
    f = ext["batch"].features_from_frame(frame, tlbr).cpu().numpy()
    crops = [frame[int(b[1]):int(b[3]), int(b[0]):int(b[2])] for b in tlbr]
    with torch.no_grad():
        exp = R.forward(sd, R.preprocess(crops), batch_stats=True).numpy()
    assert (f * exp).sum(1).min() > 0.9999 and np.abs(f - exp).max() < 2e-3


def test_features_from_frame_refuses_negative_coordinates(extractors):
    """The reference's slice ori_img[int(y1):int(y2), int(x1):int(x2)] wraps a negative coordinate to the far side of the frame; both
    branches of the drop-in get_feature refuse such boxes instead of silently cropping something else."""
    _, ext = extractors
    frame = np.zeros((100, 120, 3), np.uint8)
    with pytest.raises(L.B2TError, match="negative"):
        ext["batch"].features_from_frame(frame, np.array([[-3.0, 5.0, 40.0, 60.0]]))
    with pytest.raises(L.B2TError, match="negative"):
        ext["batch"].features_from_frame(frame, np.array([[3.0, -1.5, 40.0, 60.0]]))
    f = ext["batch"].features_from_frame(frame, np.array([[-0.5, -0.9, 40.0, 60.0]]))          # int() truncates toward 0: a valid crop
    assert f.shape == (1, 512)


def test_dropin_get_feature_generic_callable_refuses_negative_coordinates():
    """The other branch of the drop-in BoTSORT.get_feature (any reid_model(list_of_crops) callable) refuses the same boxes, and cuts
    the reference's crops otherwise."""
    pkg = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "yolov7-tracker_b200")
    saved = {k: sys.modules.pop(k) for k in list(sys.modules) if k in ("basetrack", "botsort", "matching", "kalman_filter")}
    sys.path.insert(0, os.path.join(pkg, "tracker"))
    try:
        from botsort import BoTSORT

        class Stub:
            reid_model = staticmethod(lambda crops: [c.shape for c in crops])
        frame = np.zeros((100, 120, 3), np.uint8)
        assert BoTSORT.get_feature(Stub(), np.array([[2.7, 0.5, 40.2, 60.9], [-0.5, 3.0, 120.0, 100.0]]), frame) == [(60, 38, 3), (97, 120, 3)]
        with pytest.raises(L.B2TError, match="negative"):
            BoTSORT.get_feature(Stub(), np.array([[-3.0, 5.0, 40.0, 60.0]]), frame)
    finally:
        sys.path.remove(os.path.join(pkg, "tracker"))
        for k in ("basetrack", "botsort", "matching", "kalman_filter"):
            sys.modules.pop(k, None)
        sys.modules.update(saved)
