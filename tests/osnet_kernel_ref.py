"""TEST INFRASTRUCTURE: float64 references, error bounds and runners for the OSNet kernels of csrc/b2t_osnet.cu, shared by the GPU
tier (tests/test_gpu_osnet.py) and the CPU tier (tests/test_hostsim_osnet.py, the same source under the host simulator).  16-bit values
travel as uint16 bit patterns; `dt` is "fp16" or "bf16".

Every bound is derived, not fitted: a kernel rounds its fp32 result once to the 16-bit type (at most one spacing of that type at the
result, `ulp16`) and accumulates K products in fp32 with fmaf, which errs by at most K * 2^-24 times the sum of the products' absolute
values (`S`, computed in float64 on |weights| and |inputs|).  Where a result feeds a nonlinearity (sigmoid, ReLU, max, mean) the bound
is carried through its Lipschitz constant (1/4 for the sigmoid, 1 for the others)."""
import ctypes as C

import numpy as np

from reid_kernel_ref import CODE, MEAN, STD, crop_taps, round16, ulp16, widen16  # noqa: F401

U32 = 2.0 ** -24
NAN16 = 0xFFFF                 # a NaN in both fp16 and bf16
SENT = 0x7777                  # sentinel around every output slice
PAD = 64                       # sentinel elements before and after an output


def assert_bound(got, ref, bound, what):
    got, ref, bound = np.asarray(got, np.float64), np.asarray(ref, np.float64), np.asarray(bound, np.float64)
    err = np.abs(got - ref)
    bad = ~(err <= bound)                     # NaN fails
    if bad.any():
        k = np.flatnonzero(bad.reshape(-1))[:5]
        raise AssertionError("%s: %d of %d beyond the bound, e.g. got %s ref %s bound %s" % (
            what, int(bad.sum()), bad.size, got.reshape(-1)[k], ref.reshape(-1)[k], np.broadcast_to(bound, ref.shape).reshape(-1)[k]))
    return float(np.max(err / np.maximum(bound, 1e-300))) if err.size else 0.0


def check16(got_bits, ref, s_bound, dt, what):
    """got: 16-bit result; ref: float64; s_bound: the fp32 accumulation part of the bound (before the one rounding)."""
    return assert_bound(widen16(got_bits, dt), ref, ulp16(np.abs(ref) + s_bound, dt) + s_bound, what)


# ---------------------------------------------------------------- references

def crop_ref(win, oh, ow):
    """(h, w, 3) uint8 window -> (oh, ow, 3) float64: / 255, bilinear to ow x oh with the float32 taps, Normalize."""
    a = win.astype(np.float64) / 255.0
    x0, x1, fx = crop_taps(ow, a.shape[1])
    y0, y1, fy = crop_taps(oh, a.shape[0])
    fx = fx[None, :, None]; fy = fy[:, None, None]
    rows = a[:, x0] * (1 - fx) + a[:, x1] * fx
    r = rows[y0] * (1 - fy) + rows[y1] * fy
    return (r - MEAN.astype(np.float64)) / STD.astype(np.float64)


CROP_S = 16 * U32 * 3.0        # ~12 float32 operations on values below 3 (|(v - mean) / std| < 2.7)


def _t(a):
    import torch
    return torch.from_numpy(np.ascontiguousarray(a, np.float64))


def stem_ref(x, wt, bias, drop_tap=None):
    """x (n, h, w, >= 3) float64 -> (ref, S) of the pooled (n, h/4, w/4, 16) map.  wt [(ky * 7 + kx) * 3 + ci][16]."""
    import torch.nn.functional as F
    w = _t(wt).reshape(7, 7, 3, 16).permute(3, 2, 0, 1).contiguous()
    if drop_tap is not None:
        w[:, :, drop_tap[0], drop_tap[1]] = 0
    xi = _t(x[..., :3]).permute(0, 3, 1, 2)
    y = F.relu(F.conv2d(xi, w, _t(bias), 2, 3))
    s = F.conv2d(xi.abs(), w.abs(), _t(np.abs(bias)), 2, 3)
    ref = F.max_pool2d(y, 3, 2, 1).permute(0, 2, 3, 1).numpy()
    return ref, F.max_pool2d(s, 3, 2, 1).permute(0, 2, 3, 1).numpy() * 150 * U32


def pointwise_ref(xa, xb, wt, bias, res, relu, pool):
    """float64 inputs (n, h, w, c) -> (ref, S)"""
    ca = xa.shape[-1]
    y = xa @ wt[:ca].astype(np.float64) + bias.astype(np.float64)
    s = np.abs(xa) @ np.abs(wt[:ca]).astype(np.float64) + np.abs(bias).astype(np.float64)
    k = ca
    if xb is not None:
        y = y + xb @ wt[ca:].astype(np.float64)
        s = s + np.abs(xb) @ np.abs(wt[ca:]).astype(np.float64)
        k += xb.shape[-1]
    if res is not None:
        y, s = y + res, s + np.abs(res)
    if relu:
        y = np.maximum(y, 0)
    s = s * (k + 4) * U32
    if pool:
        n, h, w, c = y.shape
        y = y.reshape(n, h // 2, 2, w // 2, 2, c).mean((2, 4))
        s = s.reshape(n, h // 2, 2, w // 2, 2, c).mean((2, 4)) + 4 * U32 * np.abs(y)
    return y, s


def lightconv_ref(x, w1, dw, bias, round_t=None):
    """x (n, h, w, c) float64 -> (ref, S).  round_t: a 16-bit type to round the 1 x 1 output to (a bug the tests inject)."""
    import torch.nn.functional as F
    c = x.shape[-1]
    t = x @ w1.astype(np.float64)
    ta = np.abs(x) @ np.abs(w1).astype(np.float64)
    if round_t is not None:
        t = widen16(round16(t, round_t), round_t)
    k = _t(dw).reshape(3, 3, c).permute(2, 0, 1)[:, None].contiguous()
    conv = lambda a, kk: F.conv2d(_t(a).permute(0, 3, 1, 2), kk, None, 1, 1, 1, c).permute(0, 2, 3, 1).numpy()   # noqa: E731
    y = np.maximum(conv(t, k) + bias.astype(np.float64), 0)
    s = (conv(ta, k.abs()) + np.abs(bias).astype(np.float64)) * (c + 12) * U32
    return y, s


def sigmoid(v):
    return 1.0 / (1.0 + np.exp(-v))


def gate_ref(streams, fc1_w, fc1_b, fc2_w, fc2_b, shared=True):
    """streams: 4 x (n, hw, c) float64 -> (ref, S, gates (4, n, c)).  shared=False: stream s uses the gate of stream 0's pooled vector
    for s = 0 and its own weights otherwise -- a stand-in for 'one gate per stream' the tests inject."""
    hw, c = streams[0].shape[1], streams[0].shape[2]
    hid = fc1_w.shape[0]
    gates, dg = [], []
    for s, x in enumerate(streams):
        p = x.mean(1)
        h = np.maximum(p @ fc1_w.T.astype(np.float64) + fc1_b, 0)
        g = sigmoid(h @ fc2_w.T.astype(np.float64) + fc2_b)
        if not shared and s > 0:
            g = sigmoid(h @ (fc2_w.T.astype(np.float64) * (1 + 0.5 * s)) + fc2_b)
        pa = np.abs(x).mean(1)
        ha = pa @ np.abs(fc1_w).T + np.abs(fc1_b)
        ga = ha @ np.abs(fc2_w).T + np.abs(fc2_b)
        gates.append(g)
        dg.append(0.25 * (hw + c + hid + 8) * U32 * ga)
    y = sum(g[:, None, :] * x for g, x in zip(gates, streams))
    s = sum(d[:, None, :] * np.abs(x) for d, x in zip(dg, streams)) + 8 * U32 * sum(g[:, None, :] * np.abs(x) for g, x in zip(gates, streams))
    return y, s, np.stack(gates)


def head_ref(x, wt, bias):
    """x (n, hw, c) float64 -> (ref, bound) of the (n, m) float32 output."""
    p = x.mean(1)
    y = np.maximum(p @ wt.astype(np.float64) + bias, 0)
    s = (np.abs(p) @ np.abs(wt).astype(np.float64) + np.abs(bias)) * (x.shape[1] + x.shape[2] + 4) * U32
    return y, s + U32 * np.abs(y)


# ---------------------------------------------------------------- inputs

def rand_weights(rng, shape, fan_in, scale=1.0):
    return (rng.normal(0, scale / np.sqrt(fan_in), shape)).astype(np.float32)


def rand_act(rng, shape, dt, relu=True):
    v = rng.normal(0.3, 1.0, shape)
    return round16(np.maximum(v, 0) if relu else v, dt)


# ---------------------------------------------------------------- runners: `be` moves arrays to the kernel's memory

def addr(be, a):
    p = be.ptr(a)
    return p.value if hasattr(p, "value") else int(p)


def _out(be, count, fill=NAN16):
    """an output of `count` 16-bit elements filled with `fill`, with PAD sentinels on each side -> (buffer, address of the output)"""
    buf = np.concatenate([np.full(PAD, SENT, np.uint16), np.full(count, fill, np.uint16), np.full(PAD, SENT, np.uint16)])
    d = be.put(buf)
    return d, addr(be, d) + 2 * PAD


def _take(be, d, count, what):
    a = be.get(d)
    assert (a[:PAD] == SENT).all() and (a[PAD + count:] == SENT).all(), "%s wrote outside its output" % what
    return a[PAD:PAD + count]


def run_crops(lib, be, buf, rows, oh, ow, dt):
    n = len(rows)
    d_buf, d_rows = be.put(buf), be.put(rows)
    d, p = _out(be, n * oh * ow * 4)
    rc = lib.b2t_osnet_crops(addr(be, d_buf), addr(be, d_rows), n, oh, ow, p, CODE[dt], be.stream())
    assert rc == 0, lib.b2t_detect_last_error()
    return _take(be, d, n * oh * ow * 4, "osnet_crops").reshape(n, oh, ow, 4)


def run_stem(lib, be, x, wt, bias, dt):
    n, h, w, pitch = x.shape
    d_x, d_w, d_b = be.put(x), be.put(wt.astype(np.float32)), be.put(bias.astype(np.float32))
    count = n * (h // 4) * (w // 4) * 16
    d, p = _out(be, count)
    rc = lib.b2t_osnet_stem(addr(be, d_x), pitch, addr(be, d_w), addr(be, d_b), n, h, w, p, CODE[dt], be.stream())
    assert rc == 0, lib.b2t_detect_last_error()
    return _take(be, d, count, "osnet_stem").reshape(n, h // 4, w // 4, 16)


def run_pointwise(lib, be, xa, xb, wt, bias, res, relu, pool, dt):
    n, h, w, ca = xa.shape
    cb = 0 if xb is None else xb.shape[-1]
    cout = wt.shape[1]
    d_xa, d_w, d_b = be.put(xa), be.put(wt.astype(np.float32)), be.put(bias.astype(np.float32))
    d_xb = None if xb is None else be.put(xb)
    d_r = None if res is None else be.put(res)
    oh, ow = (h // 2, w // 2) if pool else (h, w)
    count = n * oh * ow * cout
    d, p = _out(be, count)
    rc = lib.b2t_osnet_pointwise(addr(be, d_xa), ca, None if d_xb is None else addr(be, d_xb), cb, addr(be, d_w), addr(be, d_b),
                                 None if d_r is None else addr(be, d_r), p, n, h, w, cout, int(relu), int(pool), CODE[dt], be.stream())
    assert rc == 0, lib.b2t_detect_last_error()
    return _take(be, d, count, "osnet_pointwise").reshape(n, oh, ow, cout)


def run_lightconv(lib, be, x, w1, dw, bias, dt):
    n, h, w, c = x.shape
    d_x, d_w1, d_dw, d_b = be.put(x), be.put(w1.astype(np.float32)), be.put(dw.astype(np.float32)), be.put(bias.astype(np.float32))
    d, p = _out(be, x.size)
    rc = lib.b2t_osnet_lightconv(addr(be, d_x), addr(be, d_w1), addr(be, d_dw), addr(be, d_b), p, n, h, w, c, CODE[dt], be.stream())
    assert rc == 0, lib.b2t_detect_last_error()
    return _take(be, d, x.size, "osnet_lightconv").reshape(x.shape)


def run_gate(lib, be, streams, fc1_w, fc1_b, fc2_w, fc2_b, dt):
    n, hw, c = streams[0].shape
    ds = [be.put(s) for s in streams]
    dw = [be.put(a.astype(np.float32)) for a in (fc1_w, fc1_b, fc2_w, fc2_b)]
    d, p = _out(be, streams[0].size)
    rc = lib.b2t_osnet_gate_sum(*[addr(be, a) for a in ds], *[addr(be, a) for a in dw], p, n, hw, c, fc1_w.shape[0], CODE[dt], be.stream())
    assert rc == 0, lib.b2t_detect_last_error()
    return _take(be, d, streams[0].size, "osnet_gate_sum").reshape(streams[0].shape)


def run_head(lib, be, x, wt, bias, dt):
    n, hw, c = x.shape
    m = wt.shape[1]
    d_x, d_w, d_b = be.put(x), be.put(wt.astype(np.float32)), be.put(bias.astype(np.float32))
    out = np.full(n * m + 2 * PAD, np.nan, np.float32)
    out[:PAD] = -7.0
    out[PAD + n * m:] = -7.0
    d = be.put(out)
    rc = lib.b2t_osnet_head(addr(be, d_x), addr(be, d_w), addr(be, d_b), addr(be, d) + 4 * PAD, n, hw, c, m, CODE[dt], be.stream())
    assert rc == 0, lib.b2t_detect_last_error()
    a = be.get(d)
    assert (a[:PAD] == -7.0).all() and (a[PAD + n * m:] == -7.0).all(), "osnet_head wrote outside its output"
    return a[PAD:PAD + n * m].reshape(n, m)
