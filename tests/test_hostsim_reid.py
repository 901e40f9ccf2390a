"""not-gpu: the ReID glue kernels of csrc/b2t_reid.cu executed by the host simulator (tests/hostsim) against float64 references,
within one 16-bit ulp -- the cases of tests/test_gpu_reid_kernels.py at reduced sizes.  The simulator compiles without FMA contraction
and the nvcc build with it, so the two are compared with the reference's ulp bound, not with each other's bits.  It runs one block
at a time, so it cannot show ordering effects between blocks; the GPU tier checks those.  Also: the simulator's software fp16 / bf16
conversions against NumPy and torch."""
import ctypes as C
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.join(os.path.dirname(__file__), "hostsim"))
from simlib import sim  # noqa: E402
import reid_kernel_ref as K  # noqa: E402

DTS = ["fp16", "bf16"]
MEM = K.NumpyMem()


def _conv(fn, a, out_dtype, bf16):
    a = np.ascontiguousarray(a)
    out = np.zeros(a.shape, out_dtype)
    getattr(sim(), fn)(C.c_void_p(a.ctypes.data), C.c_void_p(out.ctypes.data), C.c_longlong(a.size), int(bf16))
    return out


@np.errstate(over="ignore", invalid="ignore")
def test_sim_fp16_conversions_match_numpy():
    bits = np.arange(65536, dtype=np.uint16)
    f = _conv("b2t_sim_from16", bits, np.float32, 0)
    ref = bits.view(np.float16).astype(np.float32)
    nan = np.isnan(ref)
    assert np.array_equal(f[~nan], ref[~nan]) and np.isnan(f[nan]).all()
    rng = np.random.default_rng(0)
    # normals, subnormals, ties, overflow to inf, the largest finite value
    v = rng.normal(0, 1, 400000) * np.exp2(rng.uniform(-27, 17, 400000))
    v = np.concatenate([v, ref[~nan].astype(np.float64) + np.exp2(np.floor(np.log2(np.abs(ref[~nan]) + 1e-30)) - 11),     # exact ties
                        [65504.0, 65519.99, 65520.0, -65520.0, 1e-8, -2.9802322387695312e-08, 2.98023223876953125e-08, 0.0, -0.0, np.inf, -np.inf]])
    v = v[np.isfinite(v) | np.isinf(v)]
    got = _conv("b2t_sim_to16", v.astype(np.float64), np.uint16, 0)
    assert np.array_equal(got, v.astype(np.float16).view(np.uint16))
    v32 = v.astype(np.float32)
    assert np.array_equal(_conv("b2t_sim_f32_to16", v32, np.uint16, 0), v32.astype(np.float16).view(np.uint16))


@np.errstate(over="ignore", invalid="ignore")
def test_sim_bf16_conversions_match_torch():
    import torch
    bits = np.arange(65536, dtype=np.uint16)
    f = _conv("b2t_sim_from16", bits, np.float32, 1)
    ref = torch.from_numpy(bits.view(np.int16)).view(torch.bfloat16).float().numpy()
    nan = np.isnan(ref)
    assert np.array_equal(f[~nan], ref[~nan]) and np.isnan(f[nan]).all()
    rng = np.random.default_rng(1)
    v32 = (rng.normal(0, 1, 400000) * np.exp2(rng.uniform(-140, 127, 400000))).astype(np.float32)
    v32 = np.concatenate([v32, ref[~nan] + np.exp2(np.floor(np.log2(np.abs(ref[~nan]) + 1e-38)) - 8).astype(np.float32),       # ties
                          np.array([3.4e38, -3.4e38, 1e-40, -1e-45, 0.0], np.float32)])
    v32 = v32[np.isfinite(v32)]
    exp = torch.from_numpy(v32).to(torch.bfloat16).view(torch.int16).numpy().view(np.uint16)
    assert np.array_equal(_conv("b2t_sim_f32_to16", v32, np.uint16, 1), exp)
    # from float64: one rounding (NumPy-side reference of the same rule, checked against torch above on float32 inputs)
    v = rng.normal(0, 1, 100000) * np.exp2(rng.uniform(-130, 120, 100000))
    assert np.array_equal(_conv("b2t_sim_to16", v, np.uint16, 1), K.round16(v, "bf16"))
    assert np.array_equal(K.round16(v32, "bf16"), exp)


@pytest.mark.parametrize("dt", DTS)
def test_sim_reid_crops_within_1ulp(dt):
    rng = np.random.default_rng(5)
    wins = [(1, 1, 4, 1, 1, 3, 1), (1, 37, 40, 0, 0, 1, 0), (45, 1, 3, 2, 0, 45, 3), (33, 20, 23, 3, 5, 40, 1),      # 1x1, 1xN, Nx1, upscale
            (128, 64, 64, 0, 2, 130, 2), (256, 128, 131, 3, 0, 256, 0), (129, 65, 70, 2, 1, 131, 1), (300, 150, 150, 0, 0, 300, 5)]
    buf, rows, contents = K.crop_frame(rng, wins)
    out = K.run_crops(sim(), MEM, buf, rows, len(wins), dt)
    for i, win in enumerate(contents):
        K.assert_within_1ulp(out[i, :, :, :3], K.crop_ref(win), dt, "crop %d %s" % (i, win.shape), floor=2.0 ** -8)
        assert (out[i, :, :, 3:] == 0).all()


@pytest.mark.parametrize("dt", DTS)
@pytest.mark.parametrize("k,h,w,c", [(3, 1, 1, 8), (3, 1, 6, 64), (3, 5, 1, 8), (3, 7, 9, 8), (3, 8, 6, 16), (2, 2, 2, 8), (2, 6, 10, 64), (3, 3, 3, 512)])
def test_sim_maxpool_exact(dt, k, h, w, c):
    rng = np.random.default_rng(h * 100 + w + c)
    x = K.round16(-np.abs(rng.normal(3, 1, (3, h, w, c))), dt)               # all negative: a padding of 0 instead of -inf shows
    got = K.run_maxpool(sim(), MEM, x, k, dt)
    assert np.array_equal(got, K.maxpool_ref(x, dt, k))


@pytest.mark.parametrize("dt", DTS)
def test_sim_add_relu_exact(dt):
    rng = np.random.default_rng(3)
    for n in (8, 8 * 37):
        a = K.rand16(rng, n, dt)
        b = K.rand16(rng, n, dt)
        b[: n // 4] = a[: n // 4] ^ np.uint16(0x8000)                           # x + (-x) = +0
        got = K.run_add_relu(sim(), MEM, a, b, dt)
        ref = K.add_relu_ref(a, b, dt)
        K.assert_within_1ulp(got, ref, dt, "add_relu n=%d" % n)
        assert np.array_equal(got, K.round16(ref, dt))                       # a float32 add of two 16-bit values rounds once, exactly
        assert (got[: n // 4] == 0).all()


@pytest.mark.parametrize("dt", DTS)
@pytest.mark.parametrize("c,n_pix,ratio,relu,inplace", [(8, 1, 0, 1, 0), (16, 7, 10, 0, 1), (32, 32, 100, 1, 1), (64, 700, 1000, 0, 0),
                                                        (128, 300, 1000, 1, 0), (256, 33, 0, 0, 0), (512, 20, 100, 1, 1), (64, 2048 * 9 + 5, 1000, 1, 0)])
def test_sim_batchnorm_within_1ulp(dt, c, n_pix, ratio, relu, inplace):
    rng = np.random.default_rng(c + n_pix)
    x, gamma, beta = K.bn_inputs(rng, n_pix + 3, c, dt, ratio)
    y, _ = K.run_bn(sim(), MEM, x, n_pix, c, gamma, beta, dt, relu, inplace)
    ref = K.bn_ref(x, dt, n_pix, c, gamma, beta, 1e-5, relu)
    K.assert_within_1ulp(y[:n_pix], ref, dt, "bn c=%d n_pix=%d mean/std=%g" % (c, n_pix, ratio))
    tail = x[n_pix:] if inplace else np.full_like(x[n_pix:], 0x7777)
    assert np.array_equal(y[n_pix:], tail), "rows past n_pix written"
    if n_pix == 1:
        assert np.array_equal(y[0], K.round16(np.maximum(beta, 0) if relu else beta, dt))


def test_sim_batchnorm_workspace_does_not_carry_over():
    rng = np.random.default_rng(11)
    x1, g1, b1 = K.bn_inputs(rng, 500, 512, "fp16", 10)
    x2, g2, b2 = K.bn_inputs(rng, 900, 64, "fp16", 100)
    ws = MEM.put(np.zeros(max(sim().b2t_batchnorm_workspace_bytes(500, 512), sim().b2t_batchnorm_workspace_bytes(900, 64)) // 8))
    K.run_bn(sim(), MEM, x1, 500, 512, g1, b1, "fp16", 0, 0, ws=ws)
    y2, _ = K.run_bn(sim(), MEM, x2, 900, 64, g2, b2, "fp16", 1, 0, ws=ws)
    y2b, _ = K.run_bn(sim(), MEM, x2, 900, 64, g2, b2, "fp16", 1, 0)
    assert np.array_equal(y2, y2b)


@pytest.mark.parametrize("dt", DTS)
@pytest.mark.parametrize("hw", [1, 32, 33])
def test_sim_avgpool_l2norm(dt, hw):
    rng = np.random.default_rng(hw)
    n = 3
    x = K.rand16(rng, (n, hw, 512), dt)
    x[1] = K.round16(np.abs(K.widen16(x[1], dt)), dt)
    x[2] = 0                                                                  # all-zero row: 0 / 0, as x.div(x.norm()) gives
    got = K.run_avgpool(sim(), MEM, x, n, hw, dt)
    ref = K.avgpool_ref(x, dt, n, hw)
    assert np.abs(got[:2] - ref[:2]).max() <= 1e-6
    assert np.isnan(got[2]).all()


def test_sim_argument_errors():
    lib = sim()
    p = C.c_void_p(16)
    assert lib.b2t_maxpool3x3s2(p, p, 1, 4, 4, 12, 1, None) != 0                 # c % 8
    assert lib.b2t_maxpool2x2s2(p, p, 1, 5, 4, 8, 1, None) != 0                  # odd side
    assert lib.b2t_maxpool2x2s2(p, p, 1, 4, 3, 8, 1, None) != 0
    assert lib.b2t_add_relu(p, p, p, 12, 1, None) != 0
    assert b"multiple of 8" in lib.b2t_detect_last_error()
    for c in (4, 12, 520, 24):                                                   # c % 8, c > 512, 256 % (c / 8) (c = 24: 3 vectors)
        assert lib.b2t_batchnorm_batch_stats(p, p, 10, c, p, p, 1e-5, 0, p, 1, None) != 0
        assert lib.b2t_batchnorm_workspace_bytes(10, c) == 0
    assert lib.b2t_batchnorm_batch_stats(p, p, 0, 64, p, p, 1e-5, 0, p, 1, None) != 0
    assert lib.b2t_avgpool_l2norm(p, p, 1, 4, 256, 1, None) != 0
    assert lib.b2t_reid_crops(p, p, 1, p, 7, None) != 0
