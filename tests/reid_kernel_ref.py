"""TEST INFRASTRUCTURE: float64 references and inputs for the ReID glue kernels of csrc/b2t_reid.cu, shared by the GPU tier
(tests/test_gpu_reid_kernels.py, nvcc build through the C ABI) and the CPU tier (tests/test_hostsim_reid.py, the same source under the
host simulator).  16-bit values travel as uint16 bit patterns; `dt` is "fp16" or "bf16".

"Within 1 ulp" means: the kernel's 16-bit result is one of the two representable neighbours of the exact (float64) result -- the value
itself when that is representable."""
import numpy as np

MANT = {"fp16": 10, "bf16": 7}
EXPB = {"fp16": 5, "bf16": 8}
MEAN = np.array([0.485, 0.456, 0.406], np.float32)          # torchvision Normalize constants, as float32 (deepsort_reid.py:128-131)
STD = np.array([0.229, 0.224, 0.225], np.float32)


def round16(v, dt):
    """float64 -> 16-bit pattern, rounded to nearest even straight from the float64 value (subnormals, overflow to inf)."""
    m, eb = MANT[dt], EXPB[dt]
    v = np.asarray(v, np.float64)
    sign = np.where(np.signbit(v), 1 << (m + eb), 0).astype(np.int64)
    inf = ((1 << eb) - 1) << m
    a = np.abs(v)
    bias = (1 << (eb - 1)) - 1
    emin = 1 - bias
    with np.errstate(all="ignore"):
        _, e = np.frexp(a)
        E = np.maximum(e.astype(np.int64) - 1, emin)
        r = np.rint(np.ldexp(a, (m - E).astype(np.int32)))
        bits = ((E + bias - 1) << m) + r.astype(np.int64)
    bits = np.where(a == 0, 0, bits)
    bits = np.where((bits >= inf) | np.isinf(a), inf, bits)
    bits = np.where(np.isnan(v), inf | (1 << (m - 1)), bits)
    return (bits | sign).astype(np.uint16)


def widen16(bits, dt):
    """16-bit pattern -> float64 (exact)."""
    m, eb = MANT[dt], EXPB[dt]
    b = np.asarray(bits, np.uint16).astype(np.int64)
    bias = (1 << (eb - 1)) - 1
    mant, ex = b & ((1 << m) - 1), (b >> m) & ((1 << eb) - 1)
    sgn = np.where((b >> (m + eb)) & 1, -1.0, 1.0)
    with np.errstate(all="ignore"):
        val = np.where(ex == 0, np.ldexp(mant.astype(np.float64), 1 - bias - m),
                       np.ldexp((mant | (1 << m)).astype(np.float64), (ex - bias - m).astype(np.int32)))
        val = np.where(ex == (1 << eb) - 1, np.where(mant == 0, np.inf, np.nan), val)
    return sgn * val


def ulp16(v, dt):
    """Spacing of the 16-bit type at |v| (the subnormal spacing below the smallest normal)."""
    m, eb = MANT[dt], EXPB[dt]
    emin = 2 - (1 << (eb - 1))
    a = np.abs(np.asarray(v, np.float64))
    with np.errstate(all="ignore"):
        E = np.where(a > 0, np.floor(np.log2(np.where(a > 0, a, 1.0))), emin)
    return np.ldexp(1.0, (np.maximum(E, emin) - m).astype(np.int32))


def ulp_error(got_bits, ref, dt):
    """|got - ref| in units of the 16-bit spacing at ref."""
    got = widen16(got_bits, dt)
    return np.abs(got - ref) / ulp16(ref, dt)


def assert_within_1ulp(got_bits, ref, dt, what="", floor=0.0):
    """Every element one of the two representable neighbours of ref.  floor > 0: below |ref| = floor the spacing at `floor` is the
    bound instead (for kernels that compute in float32 like the reference, where float32 rounding dwarfs the 16-bit spacing near 0)."""
    got_bits = np.asarray(got_bits, np.uint16)
    ref = np.asarray(ref, np.float64)
    got = widen16(got_bits, dt)
    rn_bits = round16(ref, dt)
    rn = widen16(rn_bits, dt)
    # ordered integers of the patterns: consecutive representable values differ by one (-0 and +0 both map to 0)
    order = lambda bits: np.where(bits.astype(np.int64) >> (MANT[dt] + EXPB[dt]), -1, 1) * (bits.astype(np.int64) & ((1 << (MANT[dt] + EXPB[dt])) - 1))  # noqa: E731
    o_rn, o_got = order(rn_bits), order(got_bits)
    o_other = o_rn + np.sign(ref - rn).astype(np.int64)
    ok = (o_got == o_rn) | (o_got == o_other) | (np.isnan(got) & np.isnan(ref))
    if floor > 0:
        small = np.abs(ref) < floor
        ok = np.where(small, np.abs(got - ref) <= ulp16(floor, dt), ok)
    if not ok.all():
        k = np.flatnonzero(~ok.reshape(-1))[:5]
        raise AssertionError("%s: %d of %d elements beyond 1 ulp (%s), e.g. got %s ref %s" % (
            what, int((~ok).sum()), ok.size, dt, got.reshape(-1)[k], ref.reshape(-1)[k]))
    if not ref.size:
        return 0.0
    err = np.abs(got - ref) / ulp16(np.maximum(np.abs(ref), floor), dt)       # in spacings at ref (at `floor` below it)
    return float(np.nanmax(err))


def rand16(rng, shape, dt, scale=1.0, loc=0.0):
    return round16(rng.normal(loc, scale, shape), dt)


# ---------------------------------------------------------------- b2t_reid_crops

def crop_taps(dst, src):
    """OpenCV's INTER_LINEAR rule (oracle/reid.py:_taps): float32 source coordinate, floor, edge clamp."""
    scale = np.float64(1.0) / (np.float64(dst) / np.float64(src))
    f = ((np.arange(dst, dtype=np.float64) + 0.5) * scale - 0.5).astype(np.float32)
    s = np.floor(f).astype(np.int64)
    f = (f - s.astype(np.float32)).astype(np.float32)
    lo, hi = s < 0, s >= src - 1
    f[lo] = 0; s[lo] = 0
    f[hi] = 0; s[hi] = src - 1
    return s, np.minimum(s + 1, src - 1), f.astype(np.float64)


def crop_ref(win):
    """(h, w, 3) uint8 window -> (128, 64, 3) float64: /255, bilinear to 64 x 128 with the float32 taps, Normalize."""
    a = win.astype(np.float64) / 255.0
    h, w = a.shape[:2]
    x0, x1, fx = crop_taps(64, w)
    y0, y1, fy = crop_taps(128, h)
    fx = fx[None, :, None]; fy = fy[:, None, None]
    rows = a[:, x0] * (1 - fx) + a[:, x1] * fx
    r = rows[y0] * (1 - fy) + rows[y1] * fy
    return (r - MEAN.astype(np.float64)) / STD.astype(np.float64)


def crop_cv2(win):
    """The reference's own path (Extractor._preprocess :134-146): cv2.resize on float32 / 255, then Normalize (in float64 here)."""
    import cv2
    r = cv2.resize(win.astype(np.float32) / np.float32(255.0), (64, 128)).astype(np.float64).reshape(128, 64, 3)
    return (r - MEAN.astype(np.float64)) / STD.astype(np.float64)


def crop_frame(rng, windows):
    """A uint8 buffer of frames, each holding one window (content 0..254) at (x0, y0) and sentinel 255 everywhere else, with at least
    one sentinel row before and after every frame: any read outside a window changes the output, and none leaves the buffer.
    windows: list of (h, w, pitch_px, x0, y0, frame_h, odd_lead) -> (buffer, crop rows {offset, pitch, h, w}, window contents)."""
    parts, rows, wins, off = [], [], [], 0
    for (h, w, pitch_px, x0, y0, fh, odd) in windows:
        assert x0 + w <= pitch_px and y0 + h <= fh
        frame = np.full((fh, pitch_px, 3), 255, np.uint8)
        win = rng.integers(0, 255, (h, w, 3), dtype=np.uint8)
        frame[y0:y0 + h, x0:x0 + w] = win
        lead = 3 * pitch_px + odd
        buf = np.concatenate([np.full(lead, 255, np.uint8), frame.reshape(-1), np.full(3 * pitch_px + 7, 255, np.uint8)])
        rows.append((off + lead + (y0 * pitch_px + x0) * 3, 3 * pitch_px, h, w))
        parts.append(buf)
        wins.append(win)
        off += buf.size
    return np.concatenate(parts), np.array(rows, np.int64), wins


# ---------------------------------------------------------------- pools, add + ReLU, BatchNorm, average pool + L2 norm

def maxpool_ref(x_bits, dt, k):
    """F.max_pool2d on the 16-bit values (NHWC in, NHWC out); k = 3: kernel 3, stride 2, padding 1; k = 2: kernel 2, stride 2."""
    import torch
    import torch.nn.functional as F
    x = torch.from_numpy(widen16(x_bits, dt)).permute(0, 3, 1, 2)
    y = F.max_pool2d(x, 3, 2, 1) if k == 3 else F.max_pool2d(x, 2, 2)
    return round16(y.permute(0, 2, 3, 1).numpy(), dt)


def add_relu_ref(a_bits, b_bits, dt):
    return np.maximum(widen16(a_bits, dt) + widen16(b_bits, dt), 0.0)


def bn_stats_ref(x_bits, dt, n_pix, c):
    """float64 mean and biased variance over exactly n_pix rows"""
    x = widen16(x_bits, dt).reshape(-1, c)[:n_pix]
    mean = x.mean(0)
    return mean, ((x - mean) ** 2).mean(0)


def bn_apply_ref(x_bits, dt, mean, var, gamma, beta, eps, relu):
    """scale / shift with those statistics, optional ReLU: the exact result (float64)"""
    x = widen16(x_bits, dt).reshape(-1, mean.size)
    y = (x - mean) / np.sqrt(var + np.float64(np.float32(eps))) * gamma.astype(np.float64) + beta.astype(np.float64)
    return np.maximum(y, 0.0) if relu else y


def bn_ref(x_bits, dt, n_pix, c, gamma, beta, eps, relu):
    mean, var = bn_stats_ref(x_bits, dt, n_pix, c)
    return bn_apply_ref(np.asarray(x_bits).reshape(-1, c)[:n_pix], dt, mean, var, gamma, beta, eps, relu)


def bn_inputs(rng, n_pix, c, dt, ratio):
    """x with per-channel std s in [0.5, 2] and mean = ratio * s (+-), gamma / beta near the identity."""
    s = rng.uniform(0.5, 2.0, c)
    mean = ratio * s * rng.choice([-1.0, 1.0], c)
    x = round16(rng.normal(0, 1, (n_pix, c)) * s + mean, dt)
    gamma = rng.uniform(0.5, 1.5, c).astype(np.float32)
    beta = rng.normal(0, 0.5, c).astype(np.float32)
    return x, gamma, beta


def avgpool_ref(x_bits, dt, n, hw):
    x = widen16(x_bits, dt).reshape(n, hw, 512).mean(1)
    with np.errstate(invalid="ignore"):
        return x / np.linalg.norm(x, axis=1, keepdims=True)


# ---------------------------------------------------------------- running the kernels: `be` moves arrays to the kernel's memory
class NumpyMem:
    """host simulator: device memory is host memory"""
    def put(self, a):
        return np.ascontiguousarray(a).copy()

    def ptr(self, a):
        return a.ctypes.data

    def get(self, a):
        return a

    def stream(self):
        return None


CODE = {"fp16": 1, "bf16": 0}             # B2T_ACT_F16 / B2T_ACT_BF16


def run_crops(lib, be, buf, rows, n, dt):
    """rows: (n, 4) crop rows -> (n, 128, 64, 16) uint16"""
    d_buf, d_rows = be.put(buf), be.put(rows)
    out = be.put(np.full((n, 128, 64, 16), 0x7777, np.uint16))
    rc = lib.b2t_reid_crops(be.ptr(d_buf), be.ptr(d_rows), n, be.ptr(out), CODE[dt], be.stream())
    assert rc == 0, lib.b2t_detect_last_error()
    return be.get(out)


def run_maxpool(lib, be, x, k, dt):
    n, h, w, c = x.shape
    ho, wo = ((h + 1) // 2, (w + 1) // 2) if k == 3 else (h // 2, w // 2)
    d_x = be.put(x)
    out = be.put(np.full((n, ho, wo, c), 0x7777, np.uint16))
    fn = lib.b2t_maxpool3x3s2 if k == 3 else lib.b2t_maxpool2x2s2
    rc = fn(be.ptr(d_x), be.ptr(out), n, h, w, c, CODE[dt], be.stream())
    assert rc == 0, lib.b2t_detect_last_error()
    return be.get(out)


def run_add_relu(lib, be, a, b, dt):
    d_a, d_b = be.put(a), be.put(b)
    out = be.put(np.full(a.size + 8, 0x7777, np.uint16))
    rc = lib.b2t_add_relu(be.ptr(d_a), be.ptr(d_b), be.ptr(out), a.size, CODE[dt], be.stream())
    assert rc == 0, lib.b2t_detect_last_error()
    out = be.get(out)
    assert (out[a.size:] == 0x7777).all(), "add_relu wrote past n_elems"
    return out[:a.size]


def run_bn(lib, be, x_rows, n_pix, c, gamma, beta, dt, relu, inplace, eps=1e-5, ws=None):
    """x_rows: (rows >= n_pix, c) uint16; returns all rows of y (rows past n_pix must be untouched) and the workspace used."""
    nbytes = int(lib.b2t_batchnorm_workspace_bytes(n_pix, c))
    assert nbytes > 0
    if ws is None:
        ws = be.put(np.full(nbytes // 8, np.nan, np.float64))
    d_x = be.put(x_rows)
    y = d_x if inplace else be.put(np.full(x_rows.shape, 0x7777, np.uint16))
    d_g, d_b = be.put(gamma.astype(np.float32)), be.put(beta.astype(np.float32))
    rc = lib.b2t_batchnorm_batch_stats(be.ptr(d_x), be.ptr(y), n_pix, c, be.ptr(d_g), be.ptr(d_b), eps, int(relu), be.ptr(ws), CODE[dt], be.stream())
    assert rc == 0, lib.b2t_detect_last_error()
    return be.get(y), ws


def run_avgpool(lib, be, x, n, hw, dt):
    d_x = be.put(x)
    out = be.put(np.full((n, 512), -7.0, np.float32))
    rc = lib.b2t_avgpool_l2norm(be.ptr(d_x), be.ptr(out), n, hw, 512, CODE[dt], be.stream())
    assert rc == 0, lib.b2t_detect_last_error()
    return be.get(out)
