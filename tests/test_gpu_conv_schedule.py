"""The conv kernel's consumer schedules (csrc/b2t_conv.cu): ping-pong for MT = 1 with BLOCK_N <= 128 (each consumer warpgroup owns whole
128-pixel tiles, the two take alternate tiles and alternate their MMA loops), cooperative otherwise (two warpgroups per 128-pixel
sub-tile); and the register hand-off from the producer warpgroup (setmaxnreg) that lets them hold their accumulators unspilled.

The register check needs nvcc only; the rest runs on the GPU against torch with the tolerances of test_gpu_detector.py, and checks
that every schedule gives the same bits."""
import os
import re
import shutil
import subprocess

import numpy as np
import pytest

torch = pytest.importorskip("torch")

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CONV_SRC = os.path.join(ROOT, "yolov7-tracker_b200", "csrc", "b2t_conv.cu")
NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
TOL = {torch.float16: 2e-3, torch.bfloat16: 1.5e-2}


@pytest.mark.skipif(not (os.path.exists(NVCC) or shutil.which("nvcc")), reason="nvcc not available")
def test_conv_kernel_instantiations_do_not_spill(tmp_path):
    """ptxas -v on the conv translation unit: every conv_bias_act_kernel instantiation (fp32 / 16-bit output, fp16 / bf16, mt, BLOCK_N)
    reports 0 bytes of spill stores and loads -- the consumers' accumulators fit in what the producer warpgroup hands over."""
    nvcc = NVCC if os.path.exists(NVCC) else shutil.which("nvcc")
    r = subprocess.run([nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-Xptxas", "-v", "-c", CONV_SRC,
                        "-o", str(tmp_path / "conv.o")], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-4000:]
    pat = re.compile(r"Function properties for (\S*conv_bias_act_kernelILb([01])ELb([01])ELi(\d)ELi(\d+)E\S*)\n\s*(\d+) bytes stack frame, "
                     r"(\d+) bytes spill stores, (\d+) bytes spill loads")
    found = {}
    for m in pat.finditer(r.stdout + r.stderr):
        key = (int(m.group(2)), int(m.group(3)), int(m.group(4)), int(m.group(5)))
        found[key] = (int(m.group(7)), int(m.group(8)))
    expected = {(f32, f16, mt, bn) for f32 in (0, 1) for f16 in (0, 1) for mt, bns in ((1, (32, 64, 128, 256)), (2, (32, 64, 128))) for bn in bns}
    assert set(found) == expected, "instantiations seen: %s" % sorted(found)
    spilled = {k: v for k, v in found.items() if v != (0, 0)}
    assert not spilled, "spills (stores, loads) by (f32, f16, mt, BLOCK_N): %s" % spilled


def _ref_conv(x_nhwc, w, b, stride, act):
    import torch.nn.functional as F
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    x = x_nhwc.float().permute(0, 3, 1, 2).contiguous()
    y = F.conv2d(x, w.to(x_nhwc.dtype).float(), b, stride=stride, padding=w.shape[-1] // 2)
    if act:
        y = y * torch.sigmoid(y)
    return y.permute(0, 2, 3, 1).contiguous()


PINGPONG_CASES = [
    # id, (n, h, w, cin, cout, k, s, in_pitch_extra, in_coff, out_pitch_extra, out_coff, act, f32), plan arguments
    ("flat_kpair", (2, 32, 32, 128, 128, 1, 1, 0, 0, 0, 0, True, False), dict(block_n=128, kpair=2)),
    ("flat_nokpair", (2, 32, 32, 128, 128, 1, 1, 0, 0, 0, 0, True, False), dict(block_n=64, kpair=1)),
    ("flat_bn32", (2, 24, 24, 64, 32, 1, 1, 0, 0, 0, 0, True, False), dict(block_n=32)),
    ("s2_bn128", (1, 64, 64, 64, 128, 3, 2, 0, 0, 0, 0, True, False), dict(block_n=128)),
    ("s2_bn64_tw8", (2, 48, 40, 128, 192, 3, 2, 0, 0, 0, 0, True, False), dict(block_n=64, tile_w=8)),
    ("halo_cin16", (1, 36, 24, 16, 128, 3, 1, 0, 0, 0, 0, True, False), dict(block_n=64, halo=True)),
    ("halo_cin32_bres", (2, 40, 56, 32, 64, 3, 1, 0, 0, 0, 0, True, False), dict(block_n=64, halo=True)),
    ("halo_cin192", (1, 48, 48, 192, 128, 3, 1, 0, 0, 0, 0, True, False), dict(block_n=128, halo=True)),
    ("halo_bres_64", (2, 32, 32, 64, 64, 3, 1, 0, 0, 0, 0, True, False), dict(block_n=64, halo=True)),
    ("halo_tps1", (2, 20, 20, 256, 256, 3, 1, 0, 0, 0, 0, True, False), dict(block_n=128, halo=True, tps=1)),
    ("generic_3x3", (2, 40, 40, 128, 128, 3, 1, 0, 0, 0, 0, True, False), dict(block_n=128)),
    ("head_f32", (2, 20, 20, 512, 255, 1, 1, 0, 0, 0, 0, False, True), dict(block_n=128)),
    ("head_f32_bn64", (2, 20, 20, 512, 255, 1, 1, 0, 0, 0, 0, False, True), dict(block_n=64)),
    ("concat_slices", (2, 40, 40, 128, 192, 3, 1, 64, 64, 128, 64, True, False), dict(block_n=64)),
    ("concat_slices_halo", (2, 40, 40, 128, 192, 3, 1, 64, 64, 128, 64, True, False), dict(block_n=64, halo=True)),
    ("concat_slices_flat", (2, 16, 16, 128, 64, 1, 1, 64, 64, 64, 32, True, False), dict(block_n=64)),
    # ragged tile counts on 132 SMs: 267 tiles (odd, more than 2 x grid), 201 (odd, last tile partial, between grid and 2 x grid),
    # 3 tiles (fewer than the grid could hold: warpgroup 1 of every CTA meets the terminator while warpgroup 0 has a tile)
    ("ragged_267", (1, 178, 192, 64, 64, 1, 1, 0, 0, 0, 0, True, False), dict(block_n=64)),
    ("ragged_201", (1, 100, 257, 64, 64, 1, 1, 0, 0, 0, 0, True, False), dict(block_n=64)),
    ("ragged_3", (1, 16, 24, 64, 128, 1, 1, 0, 0, 0, 0, True, False), dict(block_n=128)),
    ("ragged_halo", (3, 24, 44, 64, 128, 3, 1, 0, 0, 0, 0, True, False), dict(block_n=128, halo=True)),
    ("splitk_flat", (1, 40, 40, 1536, 384, 1, 1, 0, 0, 0, 0, True, False), dict(block_n=128, splits=3)),
    ("splitk_3x3", (2, 20, 20, 512, 256, 3, 1, 0, 0, 0, 0, True, False), dict(block_n=64, splits=4)),
    ("splitk_halo", (2, 20, 20, 512, 128, 3, 1, 0, 0, 0, 0, True, False), dict(block_n=128, splits=2, halo=True)),
]


@pytest.mark.gpu
@pytest.mark.parametrize("dt", [torch.float16, torch.bfloat16], ids=["fp16", "bf16"])
@pytest.mark.parametrize("case", PINGPONG_CASES, ids=[c[0] for c in PINGPONG_CASES])
def test_conv_pingpong_vs_torch(case, dt):
    """Ping-pong plans (MT = 1, BLOCK_N <= 128) over every addressing mode against torch; untouched concat channels stay untouched,
    and a second and third launch (tile counters, split-K flags and turn barriers start afresh) give the same bits."""
    from b200track.conv import ConvPlan, pack_conv_weight
    name, geo, extra = case
    n, h, w, cin, cout, k, s, ipx, icoff, opx, ocoff, act, f32 = geo
    g = torch.Generator(device="cuda").manual_seed(sum(map(ord, name)))
    in_pitch = cin + ipx + (icoff if ipx == 0 else 0)
    xbuf = torch.randn((n, h, w, in_pitch), device="cuda", generator=g).to(dt)
    wt = torch.randn((cout, cin, k, k), device="cuda", generator=g) * (1.5 / (cin * k * k) ** 0.5)
    bias = torch.randn(cout, device="cuda", generator=g) * 0.5
    ho, wo = (h + 2 * (k // 2) - k) // s + 1, (w + 2 * (k // 2) - k) // s + 1
    out_pitch = (cout + 7) // 8 * 8 + opx
    ybuf = torch.full((n, ho, wo, out_pitch), -77.0, device="cuda", dtype=torch.float32 if f32 else dt)
    plan = ConvPlan(xbuf, pack_conv_weight(wt, dtype=dt), bias, ybuf, n, h, w, cin, icoff, cout, k, s, ocoff, act=act, out_f32=f32, **extra)
    assert plan.info["pingpong"] == 1 and plan.info["mt"] == 1 and plan.info["splits"] == extra.get("splits", 1)
    assert plan.info["halo"] == int(extra.get("halo", False))
    plan.run()
    torch.cuda.synchronize()
    first = ybuf.clone()
    plan.run(); plan.run()
    torch.cuda.synchronize()
    assert torch.equal(first, ybuf)
    ref = _ref_conv(xbuf[..., icoff:icoff + cin], wt, bias, s, act)
    got = ybuf[..., ocoff:ocoff + cout].float()
    err = (got - ref).abs()
    assert bool((err <= TOL[dt] + TOL[dt] * ref.abs()).all()), "max err %.4g at %s" % (err.max().item(), np.unravel_index(int(err.argmax()), err.shape))
    if ocoff > 0:
        assert bool((ybuf[..., :ocoff].float() == -77.0).all())
    gran = 4 if f32 else 8
    end = ocoff + (cout + gran - 1) // gran * gran
    if out_pitch > end:
        assert bool((ybuf[..., end:].float() == -77.0).all())


@pytest.mark.gpu
@pytest.mark.parametrize("dt", [torch.float16, torch.bfloat16], ids=["fp16", "bf16"])
@pytest.mark.parametrize("k", [1, 3])
def test_conv_schedules_give_identical_bits(k, dt):
    """Ping-pong (BLOCK_N 64, 128), cooperative (BLOCK_N 256; mt = 2 with 64, 128) and, for the 3x3 layer, halo and one-tile-per-tap
    addressing all sum each output in the same K order: the outputs are equal bit for bit."""
    from b200track.conv import ConvPlan, pack_conv_weight
    g = torch.Generator(device="cuda").manual_seed(5 + k)
    n, h, w, cin, cout = 2, 40, 40, 256, 256
    x = torch.randn((n, h, w, cin), device="cuda", generator=g).to(dt)
    wt = torch.randn((cout, cin, k, k), device="cuda", generator=g) * (1.5 / (cin * k * k) ** 0.5)
    b = torch.randn(cout, device="cuda", generator=g) * 0.5
    wp = pack_conv_weight(wt, dtype=dt)
    cfgs = [dict(block_n=64), dict(block_n=128), dict(block_n=256), dict(block_n=64, mt=2), dict(block_n=128, mt=2)]
    if k == 3:
        cfgs += [dict(block_n=128, halo=True), dict(block_n=64, halo=True, mt=2), dict(block_n=256, halo=True), dict(block_n=128, tile_w=8)]
    else:
        cfgs += [dict(block_n=128, kpair=1), dict(block_n=128, kpair=2), dict(block_n=256, kpair=2)]
    outs, sched = [], []
    for cfg in cfgs:
        y = torch.zeros((n, h, w, cout), device="cuda", dtype=dt)
        plan = ConvPlan(x, wp, b, y, n, h, w, cin, 0, cout, k, 1, 0, **cfg)
        plan.run()
        outs.append(y)
        sched.append(plan.info["pingpong"])
    torch.cuda.synchronize()
    assert 0 in sched and 1 in sched
    for cfg, y in zip(cfgs[1:], outs[1:]):
        assert torch.equal(y, outs[0]), cfg
    ref = _ref_conv(x, wt, b, 1, True)
    assert bool(((outs[0].float() - ref).abs() <= TOL[dt] + TOL[dt] * ref.abs()).all())


@pytest.mark.gpu
@pytest.mark.parametrize("cfg", [dict(block_n=128), dict(block_n=64, halo=True), dict(block_n=256), dict(block_n=128, mt=2)],
                         ids=["pingpong", "pingpong_halo", "coop_bn256", "coop_mt2"])
def test_conv_back_to_back_launches_under_pdl(cfg):
    """Three launches of one plan queued back to back (programmatic dependent launch lets each start while the previous drains) give
    the bits of the first launch."""
    from b200track.conv import ConvPlan, pack_conv_weight
    dt = torch.float16
    g = torch.Generator(device="cuda").manual_seed(3)
    n, h, w, cin, cout = 4, 80, 80, 128, 256
    x = torch.randn((n, h, w, cin), device="cuda", generator=g).to(dt)
    wt = torch.randn((cout, cin, 3, 3), device="cuda", generator=g) * (1.5 / (cin * 9) ** 0.5)
    b = torch.randn(cout, device="cuda", generator=g) * 0.5
    y = torch.zeros((n, h, w, cout), device="cuda", dtype=dt)
    plan = ConvPlan(x, pack_conv_weight(wt, dtype=dt), b, y, n, h, w, cin, 0, cout, 3, 1, 0, **cfg)
    plan.run()
    torch.cuda.synchronize()
    first = y.clone()
    y.zero_()
    for _ in range(3):
        plan.run()
    torch.cuda.synchronize()
    assert torch.equal(first, y)
