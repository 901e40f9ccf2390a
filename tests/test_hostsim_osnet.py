"""not-gpu: the OSNet kernels of csrc/b2t_osnet.cu executed by the host simulator (library built by tests/hostsim/build_sim_osnet.py)
against the float64 references of tests/osnet_kernel_ref.py, at reduced sizes and with both 16-bit types; outputs start as NaN and are
fenced by sentinels.  Then the harness itself: each injected bug -- a depthwise tap dropped, one gate per stream instead of a shared one,
a nonzero halo or padding channel, H and W swapped, the 1 x 1 output rounded to 16 bits before the depthwise conv -- must fail the check
that covers it.  The simulator runs one block at a time; the GPU tier (tests/test_gpu_osnet.py) covers the full geometries."""
import os
import sys

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "hostsim"))
sys.path.insert(0, HERE)
from build_sim_osnet import sim_osnet  # noqa: E402
import osnet_kernel_ref as K  # noqa: E402
from reid_kernel_ref import NumpyMem, crop_frame  # noqa: E402

DTS = ["fp16", "bf16"]
MEM = NumpyMem()


@pytest.fixture(scope="module")
def lib():
    return sim_osnet()


@pytest.mark.parametrize("dt", DTS)
def test_sim_crops(lib, dt):
    rng = np.random.default_rng(1)
    buf, rows, wins = crop_frame(rng, [(23, 11, 40, 3, 2, 30, 1), (7, 33, 50, 10, 4, 12, 0), (1, 1, 5, 4, 0, 3, 2)])
    out = K.run_crops(lib, MEM, buf, rows, 16, 32, dt)
    for i, win in enumerate(wins):
        K.check16(out[i, ..., :3], K.crop_ref(win, 16, 32), K.CROP_S, dt, "crop %d" % i)
    assert (out[..., 3] == 0).all(), "the padding channel must be written as zero"


def _stem_case(dt, h=32, w=48, n=2, pitch=4):
    rng = np.random.default_rng(2)
    x = K.round16(rng.normal(0, 1, (n, h, w, pitch)), dt)
    x[..., 3:] = K.round16(np.full(x[..., 3:].shape, 1e3), dt)      # channels past 3 are not read
    wt = K.rand_weights(rng, (147, 16), 147)
    bias = rng.normal(0, 0.1, 16).astype(np.float32)
    return x, wt, bias


@pytest.mark.parametrize("dt", DTS)
@pytest.mark.parametrize("pitch", [4, 16])
def test_sim_stem(lib, dt, pitch):
    x, wt, bias = _stem_case(dt, pitch=pitch)
    got = K.run_stem(lib, MEM, x, wt, bias, dt)
    ref, s = K.stem_ref(K.widen16(x, dt), wt, bias)
    K.check16(got, ref, s, dt, "stem")


@pytest.mark.parametrize("dt", DTS)
@pytest.mark.parametrize("case", ["plain", "dual", "res", "pool"])
def test_sim_pointwise(lib, dt, case):
    rng = np.random.default_rng(3)
    n, h, w, ca, cb, cout = 2, 6, 10, 24, 16, 32
    xa = K.rand_act(rng, (n, h, w, ca), dt)
    xb = K.rand_act(rng, (n, h, w, cb), dt) if case == "dual" else None
    res = K.rand_act(rng, (n, h, w, cout), dt, relu=False) if case == "res" else None
    wt = K.rand_weights(rng, (ca + (cb if xb is not None else 0), cout), ca)
    bias = rng.normal(0, 0.2, cout).astype(np.float32)
    relu, pool = case != "plain", case == "pool"
    got = K.run_pointwise(lib, MEM, xa, xb, wt, bias, res, relu, pool, dt)
    W = lambda a: None if a is None else K.widen16(a, dt)       # noqa: E731
    ref, s = K.pointwise_ref(W(xa), W(xb), wt, bias, W(res), relu, pool)
    K.check16(got, ref, s, dt, "pointwise " + case)


def test_sim_pointwise_odd_pixel_count(lib):
    """n * h * w not a multiple of 4: the last quad is partial"""
    rng = np.random.default_rng(4)
    xa = K.rand_act(rng, (1, 3, 5, 16), "fp16")
    wt = K.rand_weights(rng, (16, 24), 16)
    bias = np.zeros(24, np.float32)
    got = K.run_pointwise(lib, MEM, xa, None, wt, bias, None, True, False, "fp16")
    ref, s = K.pointwise_ref(K.widen16(xa, "fp16"), None, wt, bias, None, True, False)
    K.check16(got, ref, s, "fp16", "pointwise 15 pixels")


def _light_case(dt, n=2, h=10, w=20, c=24, seed=5):
    rng = np.random.default_rng(seed)
    x = K.rand_act(rng, (n, h, w, c), dt)
    w1 = K.rand_weights(rng, (c, c), c)
    dw = K.rand_weights(rng, (9, c), 9)
    bias = rng.normal(0, 0.2, c).astype(np.float32)
    return x, w1, dw, bias


@pytest.mark.parametrize("dt", DTS)
@pytest.mark.parametrize("geom", [(2, 10, 20, 24), (1, 8, 16, 16), (1, 3, 5, 32)])
def test_sim_lightconv(lib, dt, geom):
    x, w1, dw, bias = _light_case(dt, *geom)
    got = K.run_lightconv(lib, MEM, x, w1, dw, bias, dt)
    ref, s = K.lightconv_ref(K.widen16(x, dt), w1, dw, bias)
    K.check16(got, ref, s, dt, "lightconv %s" % (geom,))


def _gate_case(dt, n=2, hw=40, c=16, hid=1, seed=6):
    rng = np.random.default_rng(seed)
    streams = [K.rand_act(rng, (n, hw, c), dt) for _ in range(4)]
    fc1_w = K.rand_weights(rng, (hid, c), c, 2.0)
    fc1_b = rng.normal(0, 0.1, hid).astype(np.float32)
    fc2_w = K.rand_weights(rng, (c, hid), hid, 2.0)
    fc2_b = rng.normal(0, 0.1, c).astype(np.float32)
    return streams, fc1_w, fc1_b, fc2_w, fc2_b


@pytest.mark.parametrize("dt", DTS)
@pytest.mark.parametrize("geom", [(2, 40, 16, 1), (1, 33, 24, 1), (2, 7, 32, 2)])
def test_sim_gate_sum(lib, dt, geom):
    streams, *fc = _gate_case(dt, *geom)
    got = K.run_gate(lib, MEM, streams, *fc, dt)
    ref, s, _ = K.gate_ref([K.widen16(a, dt) for a in streams], *fc)
    K.check16(got, ref, s, dt, "gate_sum %s" % (geom,))


@pytest.mark.parametrize("dt", DTS)
def test_sim_head(lib, dt):
    rng = np.random.default_rng(7)
    x = K.rand_act(rng, (2, 6, 128), dt)
    wt = K.rand_weights(rng, (128, 512), 128)
    bias = rng.normal(0, 0.3, 512).astype(np.float32)
    got = K.run_head(lib, MEM, x, wt, bias, dt)
    ref, bound = K.head_ref(K.widen16(x, dt), wt, bias)
    K.assert_bound(got, ref, bound, "head")


def test_sim_argument_errors(lib):
    p = 8
    assert lib.b2t_osnet_crops(p, p, 1, 16, 16, p, 7, None) != 0
    assert lib.b2t_osnet_stem(p, 3, p, p, 1, 16, 16, p, 1, None) != 0                          # pitch not a multiple of 4
    assert lib.b2t_osnet_stem(p, 4, p, p, 1, 18, 16, p, 1, None) != 0                          # height not a multiple of 4
    assert lib.b2t_osnet_pointwise(p, 12, None, 0, p, p, None, p, 1, 4, 4, 16, 1, 0, 1, None) != 0       # ca % 8
    assert lib.b2t_osnet_pointwise(p, 16, None, 0, p, p, p, p, 1, 4, 4, 16, 1, 1, 1, None) != 0          # pool + residual
    assert lib.b2t_osnet_pointwise(p, 16, None, 0, p, p, None, p, 1, 3, 4, 16, 1, 1, 1, None) != 0       # pool, odd height
    assert lib.b2t_osnet_pointwise(p, 16, None, 8, p, p, None, p, 1, 4, 4, 16, 1, 0, 1, None) != 0       # cb without xb
    assert lib.b2t_osnet_lightconv(p, p, p, p, p, 1, 4, 4, 72, 1, None) != 0                   # c > 64
    assert lib.b2t_osnet_lightconv(p, p, p, p, p, 1, 4, 4, 16, 1, None) != 0                   # in place
    assert lib.b2t_osnet_gate_sum(p, p, p, p, p, p, p, p, p, 1, 4, 16, 0, 1, None) != 0        # hidden 0
    assert lib.b2t_osnet_head(p, p, p, p, 1, 4, 300, 512, 1, None) != 0                        # c > 256
    assert b"osnet" in lib.b2t_detect_last_error()


# ---------------------------------------------------------------- the harness catches injected bugs

def test_injected_dropped_depthwise_tap_fails(lib):
    x, w1, dw, bias = _light_case("fp16")
    got = K.run_lightconv(lib, MEM, x, w1, dw, bias, "fp16")
    dw_bad = dw.copy()
    dw_bad[4] = 0                                                  # the centre tap dropped
    ref, s = K.lightconv_ref(K.widen16(x, "fp16"), w1, dw_bad, bias)
    with pytest.raises(AssertionError):
        K.check16(got, ref, s, "fp16", "lightconv")


def test_injected_dropped_stem_tap_fails(lib):
    x, wt, bias = _stem_case("fp16")
    got = K.run_stem(lib, MEM, x, wt, bias, "fp16")
    ref, s = K.stem_ref(K.widen16(x, "fp16"), wt, bias, drop_tap=(6, 6))
    with pytest.raises(AssertionError):
        K.check16(got, ref, s, "fp16", "stem")


def test_injected_gates_not_shared_fails(lib):
    streams, *fc = _gate_case("fp16")
    got = K.run_gate(lib, MEM, streams, *fc, "fp16")
    ref, s, _ = K.gate_ref([K.widen16(a, "fp16") for a in streams], *fc, shared=False)
    with pytest.raises(AssertionError):
        K.check16(got, ref, s, "fp16", "gate_sum")


def test_injected_nonzero_halo_fails(lib):
    """a depthwise conv that padded with the border's 1 x 1 output instead of zeros"""
    x, w1, dw, bias = _light_case("fp16")
    got = K.run_lightconv(lib, MEM, x, w1, dw, bias, "fp16")
    xe = np.pad(K.widen16(x, "fp16"), ((0, 0), (1, 1), (1, 1), (0, 0)), mode="edge")
    ref, s = K.lightconv_ref(xe, w1, dw, bias)
    with pytest.raises(AssertionError):
        K.check16(got, ref[:, 1:-1, 1:-1], s[:, 1:-1, 1:-1], "fp16", "lightconv")


def test_injected_nonzero_padding_channel_fails(lib):
    """crops whose padding channel were not zero (NaN from a reused buffer) would poison a pitch-16 reader; the crop check sees it"""
    rng = np.random.default_rng(1)
    buf, rows, wins = crop_frame(rng, [(23, 11, 40, 3, 2, 30, 1)])
    out = K.run_crops(lib, MEM, buf, rows, 16, 32, "fp16")
    bad = out.copy()
    bad[..., 3] = K.NAN16
    with pytest.raises(AssertionError):
        assert (bad[..., 3] == 0).all(), "the padding channel must be written as zero"
    with pytest.raises(AssertionError):
        K.check16(bad[0], np.concatenate([K.crop_ref(wins[0], 16, 32), np.zeros((16, 32, 1))], -1), K.CROP_S, "fp16", "crop")


def test_injected_swapped_sides_fails(lib):
    rng = np.random.default_rng(1)
    buf, rows, wins = crop_frame(rng, [(23, 11, 40, 3, 2, 30, 1)])
    out = K.run_crops(lib, MEM, buf, rows, 16, 32, "fp16")
    with pytest.raises(AssertionError):
        K.check16(out[0, ..., :3], K.crop_ref(wins[0], 32, 16).transpose(1, 0, 2), K.CROP_S, "fp16", "crop")


def test_injected_rounded_pointwise_before_depthwise_fails(lib):
    """the 1 x 1 output rounded to fp16 before the depthwise conv: the kernel keeps it in fp32, the bound tells the two apart"""
    x, w1, dw, bias = _light_case("fp16", c=32, seed=9)
    got = K.run_lightconv(lib, MEM, x, w1, dw, bias, "fp16")
    xw = K.widen16(x, "fp16")
    ref_exact, s = K.lightconv_ref(xw, w1, dw, bias)
    K.check16(got, ref_exact, s, "fp16", "lightconv")
    ref_round, _ = K.lightconv_ref(xw, w1, dw, bias, round_t="fp16")
    with pytest.raises(AssertionError):
        K.check16(got, ref_round, s, "fp16", "lightconv")
