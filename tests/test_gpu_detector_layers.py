"""-m gpu: every launch of the w6 and tiny forwards checked against float64, each layer from its own stored inputs
(tests/detector_layer_ref.py), at the benchmark configuration and at the shapes users run; the layer buffers bit-identical across
plans, graph replay and eager runs; and the conv epilogue swept over every finite 16-bit input.

Chain check: every layer buffer is filled with a NaN sentinel before the first run (except the zero padding of the stem input), frame
A runs, then a different frame B, and every launch is checked on B -- a tile that was never written, or that still holds frame A's
values, fails the layer it belongs to.  The per-layer table (largest err / bound, share of elements equal to the correctly rounded
float64 value, sign-normalised mean error in ulps) is printed for every configuration.

Epilogue (ConvPlan, 1x1, Cin 16, weight 1 on channel 0, so the pre-activation is the input itself): linear, ReLU and LeakyReLU are
bitwise round-to-nearest of the fp32 formula; SiLU (one tanh.approx.f32) stays within 1/2 ulp16 + 1e-5 of float64.  Largest error per
octave of the pre-activation x, measured on an H100 80GB HBM3 (700 W limit) over every finite 16-bit value and 2^18 points of [-16, 16]:
    |x| in                        [0.5, 1)  [1, 2)   [2, 4)   [4, 8)   [8, 16)  [16, 32)
    fp32 out, |error|, x < 0      7.0e-7    6.2e-6   9.0e-6   5.2e-6   9.8e-6   1.8e-6
    fp32 out, |error|, x > 0      7.0e-7    6.2e-6   9.1e-6   5.4e-6   1.02e-5  1.8e-6
    fp32 out, relative, x < 0     2.6e-5    8.0e-5   1.8e-4   1.8e-4   0.32     1 (tanh saturates at -1 below x = -16.6: output 0)
    fp16 out, ulps, x < 0         0.50      0.54     0.62     0.79     19.6     30.2
    bf16 out, ulps, x < 0         0.50      0.50     0.51     0.53     77       255
    fp16 / bf16 out, ulps, x > 0  <= 0.505 everywhere
Below |x| = 0.5 every output is within 1/2 ulp.  The epilogue's largest error, 1.02e-5 at x = 8.745, is 2 % over the 1e-5 the kernel's
comment rounds it to; the 16-bit outputs stay inside 1/2 ulp16 + 1e-5 at every input swept, which is the bar the per-layer checks use.
"""
import os
import sys
import time

import pytest

pytestmark = pytest.mark.gpu
torch = pytest.importorskip("torch")

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import detector_layer_ref as R  # noqa: E402

NAN = float("nan")


def _frames(B, H, W):
    a = torch.rand((B, 3, H, W), generator=torch.Generator().manual_seed(11)).cuda()
    b = torch.rand((B, 3, H, W), generator=torch.Generator().manual_seed(12)).cuda()
    return a, b


def _buffers(det):
    out = {}
    for buf, _ in det.place.values():
        out[buf.data_ptr()] = buf
    for t in det.spp_tmp.values():
        out.update({v.data_ptr(): v for v in t.values()})
    out.update({r.data_ptr(): r for r in det.raw})
    out[det.pred.data_ptr()] = det.pred
    return out


def _fill_sentinel(det):
    stem = det.place[0][0]
    for buf in _buffers(det).values():
        if buf is stem and det.stem_padded:
            buf[:, :, 1:1 + det.W // 2, :].fill_(NAN)                   # the zero pixel left of every row and the right padding stay
        else:
            buf.fill_(NAN)
    torch.cuda.synchronize()


def _splits(det):
    return max(p.info["splits"] for p in det.keep if hasattr(p, "info"))


def _graph(name):
    from b200track import tiny, w6
    if name == "w6":
        return w6.w6_layers(), "silu", w6.ANCHORS, w6.STRIDES, 0
    return tiny.tiny_layers(), "leaky", tiny.ANCHORS, tiny.STRIDES, -1


_SD = {}


def _sd(name):
    if name not in _SD:
        from b200track import tiny, w6
        _SD[name] = w6.calibrated_state_dict(0, 1280, "cuda", act_std=1.0) if name == "w6" else {k: v.cuda() for k, v in tiny.seeded_state_dict(0).items()}
    return _SD[name]


def _make(name, B, hw, **kw):
    from b200track.detector import DetectorW6
    from b200track.tiny import DetectorTiny
    return (DetectorW6 if name == "w6" else DetectorTiny)(_sd(name), batch=B, img_size=hw, **kw)


def _run_a_then_b(det, B, H, W):
    fa, fb = _frames(B, H, W)
    _fill_sentinel(det)
    det.forward(fa)
    det.forward(fb)
    torch.cuda.synchronize()
    return fb


def _check(name, det, img, images, title):
    layers, act, anchors, strides, no_ = _graph(name)
    views = R.detector_views(det, layers)
    t0 = time.time()
    rows = R.check_chain(layers, _sd(name), act, det.act_dtype, img, views.__getitem__, anchors, strides, images=images,
                         name_offset=no_, splits=_splits(det), pred=det.pred)
    torch.cuda.synchronize()
    print("\n" + R.format_table(rows, "%s  (float64 check of images %s: %.1f s)" % (title, images, time.time() - t0)))
    bad = R.failures(rows)
    assert not bad, "layers over their bound or not finite:\n" + R.format_table(bad)
    return rows


# ---------------------------------------------------------------- the benchmark configuration: w6, 1280^2, batch 8, fp16, autotuned, CUDA graph

@pytest.fixture(scope="module")
def bench_w6():
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    det = _make("w6", 8, 1280, act_dtype=torch.float16, autotune=True, use_graph=True)
    img = _run_a_then_b(det, 8, 1280, 1280)
    yield det, img
    del det
    torch.cuda.empty_cache()


def test_w6_1280_b8_bench_config_every_launch_vs_float64(bench_w6):
    """all eight images, one at a time (0.72 TFLOP of float64 convs per image: the reference and the |w|.|x| pass)"""
    det, img = bench_w6
    _check("w6", det, img, None, "w6 1280x1280 b8 fp16, autotuned, CUDA graph, frame B after A")


def _snapshot_equal(det_a, det_b, layers):
    va, vb = R.detector_views(det_a, layers), R.detector_views(det_b, layers)
    diff = [k for k in va if not torch.equal(va[k], vb[k])]
    return diff


def test_w6_1280_b8_bit_identical_across_plans_graph_and_eager(bench_w6):
    """the autotuned graph replay of B after A, an untuned eager run of B alone, and an eager run of B with plans tuned afresh (the
    process-wide tuning cache cleared) store the same bits in every layer buffer and in the raw head maps"""
    from b200track import detector as D
    det, img = bench_w6
    layers = _graph("w6")[0]
    eager = _make("w6", 8, 1280, act_dtype=torch.float16, autotune=False, use_graph=False)
    eager.forward(img)
    torch.cuda.synchronize()
    diff = _snapshot_equal(det, eager, layers)
    del eager
    assert not diff, "untuned eager run differs from the tuned graph replay in %s" % diff
    saved = dict(D._TUNE_CACHE)
    D._TUNE_CACHE.clear()
    try:
        retuned = _make("w6", 8, 1280, act_dtype=torch.float16, autotune=True, use_graph=False)
    finally:
        D._TUNE_CACHE.clear()
        D._TUNE_CACHE.update(saved)
    changed = [k for k in retuned.tuned if {a: b for a, b in retuned.tuned[k].items() if a != "us"} != {a: b for a, b in det.tuned.get(k, {}).items() if a != "us"}]
    retuned.forward(img)
    torch.cuda.synchronize()
    diff = _snapshot_equal(det, retuned, layers)
    print("\nretuned plans that differ from the first tuning: %d of %d convs" % (len(changed), len(retuned.tuned)))
    del retuned
    assert not diff, "eager run with freshly tuned plans differs in %s" % diff


# ---------------------------------------------------------------- the other shapes users run

@pytest.mark.parametrize("case", [
    ("w6", 2, (768, 1280), torch.bfloat16, False, False),      # a letterboxed 1080p frame (stride-64 minimum rectangle), bf16, default plans
    ("w6", 2, (192, 320), torch.float16, False, False),        # maps down to 3 x 5
    ("tiny", 1, (1280, 1280), torch.float16, True, True),      # YOLOv7-tiny as the sub-benchmark runs it
], ids=["w6-768x1280-b2-bf16", "w6-192x320-b2", "tiny-1280-b1-tuned-graph"])
def test_every_launch_vs_float64(case):
    name, B, (H, W), dt, tune, graph = case
    det = _make(name, B, (H, W), act_dtype=dt, autotune=tune, use_graph=graph)
    img = _run_a_then_b(det, B, H, W)
    _check(name, det, img, None, "%s %dx%d b%d %s autotune=%s graph=%s, frame B after A" % (name, H, W, B, dt, tune, graph))


# ---------------------------------------------------------------- epilogue sweep

def _run_1x1(x, w_rows, bias, act, out_f32):
    """x (1, h, w, 16) 16-bit; every output channel c = act(x . w_rows[c] + bias[c])"""
    from b200track.conv import ConvPlan, pack_conv_weight
    n, h, w, _ = x.shape
    cout = w_rows.shape[0]
    y = torch.full((n, h, w, cout), NAN, device="cuda", dtype=torch.float32 if out_f32 else x.dtype)
    plan = ConvPlan(x, pack_conv_weight(w_rows.view(cout, 16, 1, 1), dtype=x.dtype), bias.contiguous(), y, n, h, w, 16, 0, cout, 1, 1, 0,
                    act=act, out_f32=out_f32)
    plan.run()
    torch.cuda.synchronize()
    return y


def _inputs(dt):
    """(hi, lo) 16-bit pairs whose sum is exact in fp32: every finite value of the type (lo = 0), and a dense sweep of [-16, 16]"""
    bits = torch.arange(-32768, 32768, dtype=torch.int32).to(torch.int16)
    every = bits.view(dt)
    every = every[torch.isfinite(every.float())]
    t = torch.linspace(-16, 16, 2 ** 18 + 1, dtype=torch.float64)
    hi = t.to(dt)
    lo = (t - hi.double()).to(dt)
    hi, lo = torch.cat([every, hi]), torch.cat([torch.zeros_like(every), lo])
    pre = hi.double() + lo.double()
    keep = pre.float().double() == pre
    return hi[keep], lo[keep], pre[keep]


def _octave_table(x, err, tag):
    lines = ["%s: largest |error| per octave of the pre-activation x" % tag]
    ax = x.abs()
    for sign, sel in (("x < 0", x < 0), ("x > 0", x > 0)):
        for e in range(-10, 6):
            m = sel & (ax >= 2.0 ** e) & (ax < 2.0 ** (e + 1))
            if bool(m.any()):
                lines.append("  %s  |x| in [2^%d, 2^%d): %.3g" % (sign, e, e + 1, float(err[m].max())))
    return "\n".join(lines)


@pytest.mark.parametrize("dt", [torch.float16, torch.bfloat16], ids=["fp16", "bf16"])
def test_epilogue_sweep_every_activation(dt):
    hi, lo, pre = _inputs(dt)
    n = pre.numel()
    side = 256
    P = (n + side * side - 1) // (side * side) * side * side
    x = torch.zeros((P, 16), dtype=dt)
    x[:n, 0], x[:n, 1] = hi, lo
    x = x.view(1, P // side, side, 16).cuda()
    w = torch.zeros((16, 16), device="cuda")
    w[:, 0] = w[:, 1] = 1.0
    b0 = torch.zeros(16, device="cuda")
    pre32 = pre.float().cuda()
    pre64 = pre.cuda()
    silu64 = pre64 * torch.sigmoid(pre64)

    def out(act, f32):
        return _run_1x1(x, w, b0, act, f32).view(P, 16)[:n]

    # act 0 (fp32 out): exact; 2 ReLU / 3 LeakyReLU(0.1f) (16-bit out): bitwise round-to-nearest of the fp32 formula.  Every
    # disagreement is collected first, so one run reports all of them.
    problems = []
    slope = torch.tensor(0.1, dtype=torch.float32, device="cuda")
    for act, f32, want in ((0, True, pre32), (2, False, torch.clamp_min(pre32, 0).to(dt)), (3, False, torch.maximum(pre32, pre32 * slope).to(dt))):
        got = out(act, f32)
        bad = (got != want.view(-1, 1)).any(1)
        if bool(bad.any()):
            problems.append("act %d: %d inputs differ, e.g. x = %s -> %s, want %s" % (act, int(bad.sum()), pre64[bad][:4].tolist(),
                                                                                    got[bad][:4, 0].tolist(), want[bad][:4].tolist()))
    # SiLU: fp32 out (the epilogue's own error) and 16-bit out
    f = out(1, True)[:, 0].double()
    fin = torch.isfinite(silu64)
    err32 = (f - silu64).abs()
    tail = fin & (pre64 <= -1) & (silu64 != 0)
    print("\n" + _octave_table(pre64[fin], err32[fin], "SiLU epilogue, fp32 output, %s inputs" % dt))
    rel = err32 / silu64.abs().clamp_min(1e-300)
    print(_octave_table(pre64[tail], rel[tail], "SiLU epilogue, fp32 output, relative error in the negative tail"))
    print("max |error| %.3g at x = %.6g" % (float(err32[fin].max()), pre64[fin][err32[fin].argmax()].item()))
    if float(err32[fin].max()) > 1.05e-5:
        problems.append("SiLU epilogue error %.3g > 1.05e-5 at x = %s" % (float(err32[fin].max()), pre64[fin][err32[fin].argmax()].item()))
    y1 = out(1, False)[:, 0].double()
    bound = 0.5 * R.ulp(silu64.abs() + 1e-5, dt) + 1e-5
    e1 = (y1 - silu64).abs()
    print(_octave_table(pre64[fin], (e1 / R.ulp(silu64.abs(), dt))[fin], "SiLU, %s output, error in output ulps" % dt))
    over = fin & ~(e1 <= bound)
    if bool(over.any()):
        problems.append("SiLU beyond 1/2 ulp + 1e-5 at %d inputs, e.g. x = %s" % (int(over.sum()), pre64[over][:8].tolist()))
    # bias-only: x = 0, the pre-activation is the fp32 bias
    bias = torch.cat([torch.linspace(-16, 16, 4093, dtype=torch.float32), torch.tensor([0.0, 2.0 ** -20, -2.0 ** -20])]).cuda()
    z = torch.zeros((1, 8, 16, 16), dtype=dt, device="cuda")
    for lo_c in range(0, bias.numel(), 1024):
        bb = bias[lo_c:lo_c + 1024]
        wz = torch.zeros((bb.numel(), 16), device="cuda")
        for act, f32, want in ((0, True, bb), (2, False, torch.clamp_min(bb, 0).to(dt)), (3, False, torch.maximum(bb, bb * slope).to(dt))):
            got = _run_1x1(z, wz, bb, act, f32)
            if not torch.equal(got, want.view(1, 1, 1, -1).expand_as(got)):
                problems.append("bias-only act %d differs" % act)
        yb1 = _run_1x1(z, wz, bb, 1, False).double()
        b64 = bb.double()
        s64 = (b64 * torch.sigmoid(b64)).view(1, 1, 1, -1)
        if not bool(((yb1 - s64).abs() <= 0.5 * R.ulp(s64.abs() + 1e-5, dt) + 1e-5).all()):
            problems.append("bias-only SiLU beyond 1/2 ulp + 1e-5")
    assert not problems, "\n".join(problems)
