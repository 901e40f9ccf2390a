"""-m gpu: detector kernels (wgmma conv + bias + SiLU ...) against a plain PyTorch fp32 reference of the
same op on the same 16-bit-rounded operands, for both activation types (fp16 = the default, bf16).  Tolerance: output
rounding of the 16-bit type (2^-11 / 2^-8 relative) + fp32 accumulation order -> rtol = atol = 2e-3 (fp16) / 1.5e-2 (bf16)
on O(1) activations."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu
torch = pytest.importorskip("torch")

DTYPES = [torch.float16, torch.bfloat16]
TOL = {torch.float16: 2e-3, torch.bfloat16: 1.5e-2}


def _ref_conv(x_nhwc, w, b, stride, act):
    import torch.nn.functional as F
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    x = x_nhwc.float().permute(0, 3, 1, 2).contiguous()
    y = F.conv2d(x, w.to(x_nhwc.dtype).float(), b, stride=stride, padding=w.shape[-1] // 2)
    if act:
        y = y * torch.sigmoid(y)
    return y.permute(0, 2, 3, 1).contiguous()


CASES = [
    # n, h, w, cin, cout, k, s, in_pitch_extra, in_coff, out_pitch_extra, out_coff, act, f32
    (2, 32, 32, 64, 64, 1, 1, 0, 0, 0, 0, True, False),
    (2, 32, 32, 64, 64, 3, 1, 0, 0, 0, 0, True, False),
    (1, 64, 64, 64, 128, 3, 2, 0, 0, 0, 0, True, False),
    (2, 40, 40, 128, 192, 3, 1, 64, 64, 128, 64, True, False),     # channel slices of concat buffers
    (1, 64, 64, 16, 64, 3, 1, 0, 0, 0, 0, True, False),            # stem: BK = 16
    (2, 20, 20, 512, 255, 1, 1, 0, 0, 0, 0, False, True),          # detect head: linear, fp32, 255 -> 256 rows, pitch 256
    (2, 20, 20, 256, 256, 3, 1, 0, 0, 0, 0, True, False),          # 20x20 map: TW = 4 tiles, partial tiles
    (2, 80, 80, 256, 256, 3, 1, 0, 0, 0, 0, True, False),
    (1, 80, 80, 512, 768, 3, 2, 0, 0, 0, 0, True, False),          # stride 2, 3 N-tiles of 256
    (1, 40, 40, 1536, 384, 1, 1, 0, 0, 0, 0, True, False),         # long K (24 chunks), BN 192 x 2
]


@pytest.mark.parametrize("dt", DTYPES, ids=["fp16", "bf16"])
@pytest.mark.parametrize("case", CASES)
def test_conv_bias_silu_vs_torch(case, dt):
    from b200track.conv import ConvPlan, pack_conv_weight
    n, h, w, cin, cout, k, s, ipx, icoff, opx, ocoff, act, f32 = case
    g = torch.Generator(device="cuda").manual_seed(hash(case) % (2 ** 31))
    dev = "cuda"
    in_pitch = cin + ipx + (icoff if ipx == 0 else 0)
    xbuf = (torch.randn((n, h, w, in_pitch), device=dev, generator=g) * 1.0).to(dt)
    wt = torch.randn((cout, cin, k, k), device=dev, generator=g) * (1.5 / (cin * k * k) ** 0.5)
    bias = torch.randn(cout, device=dev, generator=g) * 0.5
    ho, wo = (h + 2 * (k // 2) - k) // s + 1, (w + 2 * (k // 2) - k) // s + 1
    out_pitch = (cout + 7) // 8 * 8 + opx
    ybuf = torch.full((n, ho, wo, out_pitch), -77.0, device=dev, dtype=torch.float32 if f32 else dt)
    plan = ConvPlan(xbuf, pack_conv_weight(wt, dtype=dt), bias.contiguous(), ybuf, n, h, w, cin, icoff, cout, k, s, ocoff, act=act, out_f32=f32)
    plan.run()
    torch.cuda.synchronize()
    ref = _ref_conv(xbuf[..., icoff:icoff + cin], wt, bias, s, act)
    got = ybuf[..., ocoff:ocoff + cout].float()
    err = (got - ref).abs()
    tol = TOL[dt] + TOL[dt] * ref.abs()
    assert bool((err <= tol).all()), "max err %.4g at %s (ref %.4g)" % (err.max().item(), np.unravel_index(int(err.argmax()), err.shape), ref.flatten()[int(err.argmax())].item())
    # untouched channels of the concat buffer stay untouched
    if ocoff > 0:
        assert bool((ybuf[..., :ocoff].float() == -77.0).all())
    # TMA stores clip at 16-byte granularity: a slice whose channel count is not a multiple of 8 (bf16) / 4 (fp32)
    # owns the padding up to the next granule (the 255-channel head owns channel 255 of its 256-wide buffer)
    gran = 4 if f32 else 8
    end = ocoff + (cout + gran - 1) // gran * gran
    if out_pitch > end:
        assert bool((ybuf[..., end:].float() == -77.0).all())


MT_CASES = [
    # n, h, w, cin, cout, k, s, block_n, mt, splits, producers
    (2, 32, 32, 128, 128, 1, 1, 128, 2, 1, 2),                    # flat: one 256-pixel A box, two MMAs per weight tile
    (1, 24, 20, 256, 192, 1, 1, 64, 2, 1, 1),                     # flat, 480 pixels: the last tile's second sub-tile is out of range
    (1, 64, 64, 64, 128, 3, 2, 128, 2, 1, 2),                     # stride 2: 16 x 16 output pixels per tile (two stacked sub-tiles)
    (2, 40, 40, 128, 128, 3, 1, 64, 2, 1, 2),                     # generic 3x3 (one tile per tap), ragged 40 = 2.5 tiles
    (1, 40, 40, 1536, 384, 1, 1, 128, 1, 3, 2),                   # split-K 3 over 24 chunks, fp32 partials reduced by the last CTA
    (2, 20, 20, 512, 512, 3, 1, 128, 1, 4, 2),                    # split-K 4 over 72 K steps
    (2, 20, 20, 512, 256, 3, 1, 64, 2, 2, 1),                     # split-K with two sub-tiles
    (1, 64, 64, 16, 64, 3, 1, 64, 2, 1, 2),                       # BK = 16 (32-byte swizzle) with two sub-tiles
]


@pytest.mark.parametrize("dt", DTYPES, ids=["fp16", "bf16"])
@pytest.mark.parametrize("case", MT_CASES)
def test_conv_subtiles_splitk_producers_vs_torch(case, dt):
    """The tiling modes of round 2 -- two 128-pixel sub-tiles per tile, split-K with a deterministic last-arriver reduction, one or
    two TMA producer warps -- against torch; split-K results must not depend on which CTA reduces (two runs bit-identical)."""
    from b200track.conv import ConvPlan, pack_conv_weight
    n, h, w, cin, cout, k, s, bn, mt, splits, prod = case
    g = torch.Generator(device="cuda").manual_seed(hash(case) % (2 ** 31))
    xbuf = torch.randn((n, h, w, cin), device="cuda", generator=g).to(dt)
    wt = torch.randn((cout, cin, k, k), device="cuda", generator=g) * (1.5 / (cin * k * k) ** 0.5)
    bias = torch.randn(cout, device="cuda", generator=g) * 0.5
    ho, wo = (h + 2 * (k // 2) - k) // s + 1, (w + 2 * (k // 2) - k) // s + 1
    ybuf = torch.full((n, ho, wo, cout), -77.0, device="cuda", dtype=dt)
    plan = ConvPlan(xbuf, pack_conv_weight(wt, dtype=dt), bias, ybuf, n, h, w, cin, 0, cout, k, s, 0, block_n=bn, mt=mt, splits=splits, producers=prod)
    assert plan.info["mt"] == mt and plan.info["splits"] == splits and plan.info["producers"] == prod
    plan.run()
    torch.cuda.synchronize()
    first = ybuf.clone()
    plan.run(); plan.run()                                            # tile counters and split-K arrival flags re-arm themselves
    torch.cuda.synchronize()
    assert torch.equal(first, ybuf)
    ref = _ref_conv(xbuf, wt, bias, s, True)
    err = (ybuf.float() - ref).abs()
    assert bool((err <= TOL[dt] + TOL[dt] * ref.abs()).all()), "max err %.4g at %s" % (err.max().item(), np.unravel_index(int(err.argmax()), err.shape))


HALO_CASES = [
    # n, h, w, cin, cout, in_pitch_extra, in_coff, out_pitch_extra, out_coff, block_n, stages
    (2, 32, 32, 64, 64, 0, 0, 0, 0, 0, 0),
    (1, 80, 80, 256, 256, 0, 0, 0, 0, 128, 3),
    (2, 20, 20, 512, 512, 0, 0, 0, 0, 64, 6),                      # 20x20: partial 16 x 8 tiles on both axes
    (2, 40, 40, 128, 192, 64, 64, 128, 64, 64, 2),                 # slices of concat buffers, 3 N tiles
    (1, 24, 44, 64, 64, 0, 0, 0, 0, 0, 0),                         # ragged: 44 = 5.5 tiles wide, 24 = 1.5 tiles high
    (1, 48, 48, 192, 256, 0, 0, 0, 0, 256, 4),                     # 3 K chunks, one 256-wide N tile
    (2, 40, 56, 32, 64, 0, 0, 0, 0, 0, 0),                         # Cin = 32: 64-byte rows, 64-byte swizzle
    (1, 36, 24, 16, 128, 0, 0, 0, 0, 64, 2),                       # Cin = 16: 32-byte rows; two N tiles, so the weights stream
]


@pytest.mark.parametrize("dt", DTYPES, ids=["fp16", "bf16"])
@pytest.mark.parametrize("mt", [1, 2])
@pytest.mark.parametrize("case", HALO_CASES)
def test_conv_halo_tile_vs_torch(case, mt, dt):
    """3x3 / stride 1 in halo-tile mode (one (16+2) x (8 mt + 2) input tile per K chunk, nine shifted shared-memory windows per
    128-pixel sub-tile) against torch on the same 16-bit-rounded operands; mt = 2: two sub-tiles side by side share every
    weight tile (shared-memory descriptors strided by an 18-pixel row pitch)."""
    from b200track.conv import ConvPlan, pack_conv_weight
    from b200track._lib import B2TError
    n, h, w, cin, cout, ipx, icoff, opx, ocoff, bn, st = case
    if 2 * mt * (bn or 128) > 512:
        x0 = torch.zeros((n, h, w, cin), device="cuda", dtype=dt); y0 = torch.zeros((n, h, w, cout), device="cuda", dtype=dt)
        with pytest.raises(B2TError):                                 # mt x BLOCK_N > 256: four consumer warpgroups' accumulators exceed the registers
            ConvPlan(x0, pack_conv_weight(torch.zeros((cout, cin, 3, 3), device="cuda"), dtype=dt), torch.zeros(cout, device="cuda"), y0, n, h, w, cin, 0,
                     cout, 3, 1, 0, block_n=bn, stages=st, halo=True, mt=mt)
        return
    g = torch.Generator(device="cuda").manual_seed(hash(case) % (2 ** 31))
    in_pitch = cin + ipx + (icoff if ipx == 0 else 0)
    xbuf = torch.randn((n, h, w, in_pitch), device="cuda", generator=g).to(dt)
    wt = torch.randn((cout, cin, 3, 3), device="cuda", generator=g) * (1.5 / (cin * 9) ** 0.5)
    bias = torch.randn(cout, device="cuda", generator=g) * 0.5
    out_pitch = cout + opx
    ybuf = torch.full((n, h, w, out_pitch), -77.0, device="cuda", dtype=dt)
    plan = ConvPlan(xbuf, pack_conv_weight(wt, dtype=dt), bias, ybuf, n, h, w, cin, icoff, cout, 3, 1, ocoff, block_n=bn, stages=st, halo=True, mt=mt)
    plan.run(); plan.run()                                            # twice: the tile counters re-arm themselves
    torch.cuda.synchronize()
    ref = _ref_conv(xbuf[..., icoff:icoff + cin], wt, bias, 1, True)
    got = ybuf[..., ocoff:ocoff + cout].float()
    err = (got - ref).abs()
    assert bool((err <= TOL[dt] + TOL[dt] * ref.abs()).all()), "max err %.4g at %s" % (err.max().item(), np.unravel_index(int(err.argmax()), err.shape))
    if ocoff > 0:
        assert bool((ybuf[..., :ocoff].float() == -77.0).all())
    if out_pitch > ocoff + cout:
        assert bool((ybuf[..., ocoff + cout:].float() == -77.0).all())


@pytest.mark.parametrize("dt", DTYPES, ids=["fp16", "bf16"])
@pytest.mark.parametrize("mode", ["rowpack", "padded_rows", "halo_mt1", "halo_mt2"])
def test_conv_stem_padded_input_vs_torch(mode, dt):
    """The w6 stem (16 -> 64, 3x3) on the padded ReOrg layout: rows of w + 8 pixels, image at pixel 1, zeros around.
    rowpack: the three kw taps of a kernel row are one 64-wide K chunk read through an overlapping-stride tensor map;
    padded_rows: the generic 9-tap addressing on the same buffer; halo_*: one (16+2) x (8 mt + 2) x 16-channel input tile
    (32-byte rows, 32-byte swizzle) feeds nine K = 16 MMAs per sub-tile, the nine 2 KB weight tiles stay resident."""
    from b200track.conv import ConvPlan, pack_conv_weight, pack_conv_weight_rowpack
    n, h, w, cout = 2, 48, 80, 64
    g = torch.Generator(device="cuda").manual_seed(77)
    row = w + 8
    xbuf = torch.zeros((n, h, row, 16), device="cuda", dtype=dt)
    xbuf[:, :, 1:w + 1, :12] = torch.randn((n, h, w, 12), device="cuda", generator=g).to(dt)
    wt = torch.zeros((cout, 16, 3, 3), device="cuda")
    wt[:, :12] = torch.randn((cout, 12, 3, 3), device="cuda", generator=g) * (1.5 / 108 ** 0.5)
    bias = torch.randn(cout, device="cuda", generator=g) * 0.5
    ybuf = torch.full((n, h, w, cout), -77.0, device="cuda", dtype=dt)
    if mode == "rowpack":
        plan = ConvPlan(xbuf, pack_conv_weight_rowpack(wt, dtype=dt), bias, ybuf, n, h, w, 16, 0, cout, 3, 1, 0, in_row_pixels=row, rowpack=True, x_pixel0=0)
    elif mode == "padded_rows":
        plan = ConvPlan(xbuf, pack_conv_weight(wt, dtype=dt), bias, ybuf, n, h, w, 16, 0, cout, 3, 1, 0, in_row_pixels=row, x_pixel0=1)
    else:
        mt = int(mode[-1])
        plan = ConvPlan(xbuf, pack_conv_weight(wt, dtype=dt), bias, ybuf, n, h, w, 16, 0, cout, 3, 1, 0, in_row_pixels=row, x_pixel0=1, halo=True, mt=mt)
        assert plan.info["halo"] == 1 and plan.info["mt"] == mt and plan.info["b_res"] == 1
    plan.run(); plan.run()
    torch.cuda.synchronize()
    ref = _ref_conv(xbuf[:, :, 1:w + 1, :], wt, bias, 1, True)
    err = (ybuf.float() - ref).abs()
    assert bool((err <= TOL[dt] + TOL[dt] * ref.abs()).all()), "max err %.4g" % err.max().item()
    assert abs(plan.flops - 2.0 * n * h * w * cout * 9 * 16) < 1.0            # algorithmic flops, not the padded K


@pytest.mark.parametrize("dt", DTYPES, ids=["fp16", "bf16"])
def test_conv_tilings_and_addressing_give_identical_bits(dt):
    """Every plan the autotuner may pick for a layer sums each output in the same order (K channel-chunk-major, taps inside), so the
    results are bit-identical whatever the tiling (BLOCK_N, sub-tiles, ring depth) and the addressing (one tile per tap, halo tile,
    row-packed stem): two independently tuned detectors compute the same detections."""
    from b200track.conv import ConvPlan, pack_conv_weight, pack_conv_weight_rowpack
    g = torch.Generator(device="cuda").manual_seed(11)
    n, h, w, cin, cout = 2, 40, 40, 192, 128
    x = torch.randn((n, h, w, cin), device="cuda", generator=g).to(dt)
    wt = torch.randn((cout, cin, 3, 3), device="cuda", generator=g) * (1.5 / (cin * 9) ** 0.5)
    b = torch.randn(cout, device="cuda", generator=g) * 0.5
    wp = pack_conv_weight(wt, dtype=dt)
    outs = []
    for cfg in (dict(), dict(block_n=128, mt=1, stages=3), dict(block_n=64, mt=2, stages=2), dict(halo=True), dict(halo=True, mt=2, block_n=64)):
        y = torch.zeros((n, h, w, cout), device="cuda", dtype=dt)
        ConvPlan(x, wp, b, y, n, h, w, cin, 0, cout, 3, 1, 0, **cfg).run()
        outs.append(y)
    # the w6 stem on the padded ReOrg layout: row-packed, nine taps, halo
    row, cs = w + 8, 64
    xs = torch.zeros((n, h, row, 16), device="cuda", dtype=dt)
    xs[:, :, 1:w + 1, :12] = torch.randn((n, h, w, 12), device="cuda", generator=g).to(dt)
    ws = torch.zeros((cs, 16, 3, 3), device="cuda")
    ws[:, :12] = torch.randn((cs, 12, 3, 3), device="cuda", generator=g) * (1.5 / 108 ** 0.5)
    bs = torch.randn(cs, device="cuda", generator=g) * 0.5
    stems = []
    for wpk, cfg in ((pack_conv_weight_rowpack(ws, dtype=dt), dict(rowpack=True, x_pixel0=0)), (pack_conv_weight(ws, dtype=dt), dict(x_pixel0=1)),
                     (pack_conv_weight(ws, dtype=dt), dict(x_pixel0=1, halo=True))):
        y = torch.zeros((n, h, w, cs), device="cuda", dtype=dt)
        ConvPlan(xs, wpk, bs, y, n, h, w, 16, 0, cs, 3, 1, 0, in_row_pixels=row, **cfg).run()
        stems.append(y)
    torch.cuda.synchronize()
    for y in outs[1:]:
        assert torch.equal(y, outs[0])
    for y in stems[1:]:
        assert torch.equal(y, stems[0])


# ------------------------------------------------------------------------------------------ glue kernels
def _lib():
    from b200track import _lib as L
    return L, L.load()


def _s():
    import ctypes as C
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


@pytest.mark.parametrize("dt", DTYPES, ids=["fp16", "bf16"])
def test_image_reorg_matches_reference_order(dt):
    import ctypes as C
    L, lib = _lib()
    code = L.act_dtype_code(dt)
    img = torch.rand((2, 3, 64, 96), device="cuda")
    out = torch.zeros((2, 32, 48, 16), dtype=dt, device="cuda")
    assert lib.b2t_image_reorg(C.c_void_p(img.data_ptr()), C.c_void_p(out.data_ptr()), 2, 64, 96, code, _s()) == 0
    ref = torch.cat([img[..., ::2, ::2], img[..., 1::2, ::2], img[..., ::2, 1::2], img[..., 1::2, 1::2]], 1)   # models/common.py:52-53
    assert torch.equal(out[..., :12].float(), ref.permute(0, 2, 3, 1).to(dt).float())
    assert bool((out[..., 12:] == 0).all())
    padded = torch.full((2, 32, 48 + 8, 16), 5.0, dtype=dt, device="cuda")
    assert lib.b2t_image_reorg_padded(C.c_void_p(img.data_ptr()), C.c_void_p(padded.data_ptr()), 2, 64, 96, 56, 1, code, _s()) == 0
    assert torch.equal(padded[:, :, 1:49], out) and bool((padded[:, :, 0] == 5.0).all()) and bool((padded[:, :, 49:] == 5.0).all())


@pytest.mark.parametrize("dt", DTYPES, ids=["fp16", "bf16"])
def test_upsample_and_spp_pool(dt):
    import ctypes as C
    import torch.nn.functional as F
    L, lib = _lib()
    src = torch.randn((2, 10, 10, 48), device="cuda").to(dt)
    dst = torch.zeros((2, 20, 20, 64), dtype=dt, device="cuda")
    assert lib.b2t_upsample2x(C.c_void_p(src.data_ptr()), 48, 16, C.c_void_p(dst.data_ptr()), 64, 32, 2, 10, 10, 32, _s()) == 0
    ref = F.interpolate(src[..., 16:48].float().permute(0, 3, 1, 2), scale_factor=2, mode="nearest").permute(0, 2, 3, 1)
    assert torch.equal(dst[..., 32:64].float(), ref) and bool((dst[..., :32] == 0).all())
    # 20 x 20 / 7 x 11: the shared-memory plane kernel; 40 x 40: plane too large -> the direct kernel; 6 channels: direct too
    for (h, w, c) in ((20, 20, 16), (7, 11, 8), (40, 40, 16), (12, 12, 6)):
        buf = torch.zeros((2, h, w, 4 * c), dtype=dt, device="cuda")
        buf[..., :c] = torch.randn((2, h, w, c), device="cuda").to(dt)
        assert lib.b2t_spp_pool(C.c_void_p(buf.data_ptr()), 4 * c, c, 2, h, w, L.act_dtype_code(dt), _s()) == 0
        x = buf[..., :c].float().permute(0, 3, 1, 2)
        for n, k in enumerate((5, 9, 13)):
            ref = F.max_pool2d(x, k, 1, k // 2).permute(0, 2, 3, 1)
            assert torch.equal(buf[..., c * (n + 1):c * (n + 2)].float(), ref), (h, w, c, k)


def test_nms_matches_reference_algorithm():
    """b2t_nms on a dense (B, N, 85) prediction == utils/general.py non_max_suppression with torchvision.ops.nms."""
    import ctypes as C
    from oracle import detector as OD
    L, lib = _lib()
    g = torch.Generator(device="cuda").manual_seed(5)
    B, N = 3, 6000
    pred = torch.zeros((B, N, 85), device="cuda")
    pred[..., 0:2] = torch.rand((B, N, 2), device="cuda", generator=g) * 600
    pred[..., 2:4] = torch.rand((B, N, 2), device="cuda", generator=g) * 120 + 8
    pred[..., 4] = torch.sigmoid(torch.randn((B, N), device="cuda", generator=g) * 1.5 - 3.0)
    pred[..., 5:] = torch.sigmoid(torch.randn((B, N, 80), device="cuda", generator=g))
    pred[2, :, 4] = 0.0                                              # an image without candidates -> (0, 6)
    max_det, max_nms = 300, 30000
    ws = torch.empty(lib.b2t_nms_workspace_bytes(B, N, max_nms), dtype=torch.uint8, device="cuda")
    out = torch.zeros((B, max_det, 6), device="cuda"); cnt = torch.zeros(B, dtype=torch.int32, device="cuda")
    rc = lib.b2t_nms(C.c_void_p(pred.data_ptr()), B, N, 85, 0.01, 0.45, max_det, max_nms, N, 0, 1.0, 0.0, 0.0, 640.0, 640.0,
                     C.c_void_p(ws.data_ptr()), ws.numel(), C.c_void_p(out.data_ptr()), C.c_void_p(cnt.data_ptr()), _s())
    assert rc == 0, lib.b2t_detect_last_error()
    ref = OD.non_max_suppression(pred.clone(), conf_thres=0.01, iou_thres=0.45)
    for b in range(B):
        n = int(cnt[b])
        assert n == ref[b].shape[0]
        if n:
            assert torch.equal(out[b, :n, 5], ref[b][:, 5])                                  # same boxes, same order
            assert torch.allclose(out[b, :n, :5], ref[b][:, :5], rtol=0, atol=1e-4)


def test_detector_w6_end_to_end_vs_oracle():
    """Full YOLOv7-w6 forward + decode + NMS at 256 x 256, batch 2, seeded weights.
    (1) against the oracle run with bf16 operand rounding (the arithmetic the tensor cores do): tight;
    (2) against the pure fp32 oracle: the detection sets agree up to bf16 noise."""
    from b200track.detector import DetectorW6
    from b200track.w6 import ANCHORS, STRIDES, seeded_state_dict, w6_layers
    from oracle import detector as OD
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    sd = seeded_state_dict(0)
    g = torch.Generator().manual_seed(321)
    img = torch.rand((2, 3, 256, 256), generator=g).cuda()
    det = DetectorW6(sd, batch=2, img_size=256, use_graph=False)
    pred = det.forward(img).clone()
    torch.cuda.synchronize()
    sd_gpu = {k: v.cuda() for k, v in sd.items()}
    with torch.no_grad():
        ref_bf, raw_bf = OD.forward(w6_layers(), sd_gpu, img, ANCHORS, STRIDES, emulate_bf16=det.act_dtype, return_raw=True)
        ref_32 = OD.forward(w6_layers(), sd_gpu, img, ANCHORS, STRIDES)
    # raw logits vs the bf16-emulating oracle
    off = 0
    for lvl, r in enumerate(raw_bf):
        got = det.raw[lvl][..., :255].reshape(2, r.shape[2], r.shape[3], 3, 85).permute(0, 3, 1, 2, 4)
        err = (got - r).abs()
        assert float(err.max()) < 0.25 and float(err.mean()) < 0.02, "level %d: max %.3f mean %.4f" % (lvl, err.max(), err.mean())
    d = (pred - ref_bf).abs()
    assert float((d[..., 4]).max()) < 0.02                          # objectness
    # decoded boxes: relative
    # boxes: wh = (2 sigmoid)^2 * anchor doubles the logit noise (bf16 rounding flips accumulate over ~60 layers)
    rel = d[..., :4] / (ref_bf[..., :4].abs() + 1.0)
    assert float(rel.max()) < 0.25 and float(rel.mean()) < 0.01
    out, cnt = det.detect(img, post=False)
    torch.cuda.synchronize()
    ref_nms = OD.non_max_suppression(pred, conf_thres=0.01)         # same pred -> NMS must agree exactly
    out, cnt = out.clone(), cnt.clone()
    out2, cnt2 = det.nms_from_pred(post=False)                      # two-step path (decode -> b2t_nms) == fused path, bit for bit
    torch.cuda.synchronize()
    assert torch.equal(cnt, cnt2)
    for b in range(2):
        n = int(cnt[b])
        assert n == ref_nms[b].shape[0] and torch.equal(out[b, :n, 5], ref_nms[b][:, 5])
        assert torch.allclose(out[b, :n, :5], ref_nms[b][:, :5], atol=1e-3)
        assert torch.equal(out[b, :n], out2[b, :n])
    # against the fp32 oracle: most detections have a partner with IoU > 0.9 and |dconf| < 0.02
    import torchvision
    ref32_nms = OD.non_max_suppression(ref_32, conf_thres=0.01)
    for b in range(2):
        n = int(cnt[b])
        if n == 0 or ref32_nms[b].shape[0] == 0:
            continue
        iou = torchvision.ops.box_iou(out[b, :n, :4], ref32_nms[b][:, :4])
        best, j = iou.max(1)
        ok = (best > 0.9) & ((out[b, :n, 4] - ref32_nms[b][j, 4]).abs() < 0.02) & (out[b, :n, 5] == ref32_nms[b][j, 5])
        assert float(ok.float().mean()) > 0.8, "only %.2f of the detections match the fp32 oracle" % float(ok.float().mean())


def test_detector_w6_full_size_tiles_vs_oracle():
    """640 x 640, batch 1, LSUV-calibrated weights: every tile shape / partial tile of the real network sizes
    (320 ... 10 px maps) against the bf16-emulating oracle, plus a sane NMS load."""
    from b200track.detector import DetectorW6
    from b200track.w6 import ANCHORS, STRIDES, calibrated_state_dict, w6_layers
    from oracle import detector as OD
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    sd = calibrated_state_dict(0, 640, "cuda")
    g = torch.Generator().manual_seed(99)
    img = torch.rand((1, 3, 640, 640), generator=g).cuda()
    det = DetectorW6(sd, batch=1, img_size=640, use_graph=True)
    out, cnt = det.detect(img, post=True)
    torch.cuda.synchronize()
    with torch.no_grad():
        ref_bf, raw_bf = OD.forward(w6_layers(), sd, img, ANCHORS, STRIDES, emulate_bf16=det.act_dtype, return_raw=True)
    for lvl, r in enumerate(raw_bf):
        got = det.raw[lvl][..., :255].reshape(1, r.shape[2], r.shape[3], 3, 85).permute(0, 3, 1, 2, 4)
        err = (got - r).abs()
        # bf16 rounding flips decorrelate the two pipelines over ~60 layers: mean |dlogit| ~ 0.03 (2 % of the logit std)
        rel_rms = float((err ** 2).mean().sqrt() / r.std())
        assert float(err.mean()) < 0.12 and rel_rms < 0.12, "level %d: max %.3f mean %.4f rel rms %.3f" % (lvl, err.max(), err.mean(), rel_rms)
    det.decode(); torch.cuda.synchronize()                           # detect() fuses the decode into NMS: materialise pred for the check
    ncand = int((det.pred[0, :, 4] > 0.01).sum())
    assert 0.01 * det.n_total < ncand < 0.3 * det.n_total, ncand
    ref = OD.post_process(OD.non_max_suppression(det.pred, conf_thres=0.01)[0], (640, 640))
    n = int(cnt[0])
    assert n == ref.shape[0] == 300                                  # the max_det cap is hit
    assert torch.equal(out[0, :n, 5], ref[:, 5]) and torch.allclose(out[0, :n, :5], ref[:, :5], atol=1e-3)
    assert bool((out[0, :n, :4] == out[0, :n, :4].round()).all())    # integer pixel boxes reach the tracker (q9)


def _kept_match(ours, ref, iou_t=0.99, dconf=1e-2):
    """SURVEY 7.2 #5: fraction of rows of `ours` with a row of `ref` of the same class at IoU >= iou_t and |dconf| <= dconf."""
    import torchvision
    if ours.shape[0] == 0 or ref.shape[0] == 0:
        return 0.0
    iou = torchvision.ops.box_iou(ours[:, :4], ref[:, :4])
    ok = (iou >= iou_t) & (ours[:, 5:6] == ref[:, 5].unsqueeze(0)) & ((ours[:, 4:5] - ref[:, 4].unsqueeze(0)).abs() <= dconf)
    return float(ok.any(1).float().mean())


@pytest.mark.parametrize("size,batch", [(640, 1), (1280, 8)], ids=["640x640-b1", "1280x1280-b8-bench-config"])
def test_detector_parity_vs_fp32_oracle_survey_criterion(size, batch):
    """SURVEY 7.2 #5 detector parity, at 640 x 640 and at the bench configuration (1280 x 1280, batch 8): the post-NMS kept set
    against the pure fp32 oracle -- same class, IoU >= 0.99, |dconf| <= 1e-2 -- in both directions, fp16 activations.

    Two weight sets, both seeded and LSUV-calibrated on the same image:
      * act_std = 0.3 (SiLU near its linear range: the random 60-layer net does NOT amplify perturbations): >= 93 % of the 300
        kept boxes per image must meet the criterion,
        raw logits within 0.2 % rms of the fp32 oracle, objectness within 5e-3;
      * act_std = 1.0, the bench weights: the network itself is chaotic there (the torch oracle with the same fp16 rounding only
        reaches 52-77 % against fp32), so the bar is the oracle's own: >= 40 % at IoU 0.99 and not more than 15 points below the
        fp16-rounding oracle, >= 80 % at IoU 0.95, logits within 0.8 % rms."""
    from b200track.detector import DetectorW6
    from b200track.w6 import ANCHORS, STRIDES, calibrated_state_dict, w6_layers
    from oracle import detector as OD
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    layers = w6_layers()
    g = torch.Generator().manual_seed(4000 + size)
    img = torch.rand((batch, 3, size, size), generator=g).cuda()
    # (the 640 x 640 bench-style weights are deeper in the chaotic regime -- the fp16-rounding oracle agrees with fp32 on 6 % of
    # the boxes there -- so the act_std = 1.0 leg runs at the bench configuration only)
    for act_std, min99, rms_max, obj_max in ((0.3, 0.93, 0.002, 5e-3),) + (((1.0, 0.40, 0.008, 0.05),) if size == 1280 else ()):
        sd = calibrated_state_dict(0, size, "cuda", act_std=act_std)
        det = DetectorW6(sd, batch=batch, img_size=size, use_graph=False, autotune=False)
        assert det.act_dtype == torch.float16
        pred = det.forward(img).clone()
        out, cnt = det.detect(img, post=False)
        torch.cuda.synchronize()
        with torch.no_grad():
            ref32, raw32 = OD.forward(layers, sd, img, ANCHORS, STRIDES, return_raw=True)
        for lvl, r in enumerate(raw32):
            got = det.raw[lvl][..., :255].reshape(batch, r.shape[2], r.shape[3], 3, 85).permute(0, 3, 1, 2, 4)
            rel = float(((got - r) ** 2).mean().sqrt() / r.std())
            assert rel < rms_max, "act_std %.1f level %d: rel rms %.4f vs the fp32 oracle" % (act_std, lvl, rel)
        assert float((pred[..., 4] - ref32[..., 4]).abs().max()) < obj_max
        nms32 = OD.non_max_suppression(ref32, conf_thres=0.01)
        emu = None
        if act_std == 1.0:
            with torch.no_grad():
                emu = OD.non_max_suppression(OD.forward(layers, sd, img, ANCHORS, STRIDES, emulate_bf16=torch.float16), conf_thres=0.01)
        for b in range(batch):
            n = int(cnt[b])
            assert n == nms32[b].shape[0] == 300                         # the cap is hit on both sides
            fwd, rev = _kept_match(out[b, :n], nms32[b]), _kept_match(nms32[b], out[b, :n])
            assert fwd >= min99 and rev >= min99, "act_std %.1f image %d: %.3f / %.3f of the kept boxes meet IoU >= 0.99, |dconf| <= 1e-2" % (act_std, b, fwd, rev)
            if emu is not None:
                assert fwd >= _kept_match(emu[b], nms32[b]) - 0.15
                assert _kept_match(out[b, :n], nms32[b], iou_t=0.95) >= 0.80
        del det
        torch.cuda.empty_cache()


def test_detector_stride_64_shapes():
    """Image sides that are multiples of the model stride 64 but not of 128 -- what check_img_size(s=64) / letterbox(stride=64)
    produce for 4:3 sources (960 x 1280) -- run like any other: 192 x 320 here (maps 96x160 ... 3x5), logits against the
    fp16-rounding oracle, NMS rows exact."""
    from b200track.detector import DetectorW6
    from b200track.w6 import ANCHORS, STRIDES, calibrated_state_dict, w6_layers
    from oracle import detector as OD
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    g = torch.Generator().manual_seed(64)
    img = torch.rand((2, 3, 192, 320), generator=g).cuda()
    sd = calibrated_state_dict(0, 320, "cuda", img=img[:1], act_std=0.5)
    det = DetectorW6(sd, batch=2, img_size=(192, 320), use_graph=False, autotune=False)
    pred = det.forward(img).clone()
    out, cnt = det.detect(img, post=True)
    torch.cuda.synchronize()
    with torch.no_grad():
        ref, raws = OD.forward(w6_layers(), sd, img, ANCHORS, STRIDES, emulate_bf16=det.act_dtype, return_raw=True)
    assert tuple(pred.shape) == tuple(ref.shape) == (2, 3 * (24 * 40 + 12 * 20 + 6 * 10 + 3 * 5), 85)
    for lvl, r in enumerate(raws):
        got = det.raw[lvl][..., :255].reshape(2, r.shape[2], r.shape[3], 3, 85).permute(0, 3, 1, 2, 4)
        assert float(((got - r) ** 2).mean().sqrt() / r.std()) < 0.01, lvl
    for b in range(2):
        exp = OD.post_process(OD.non_max_suppression(pred, conf_thres=0.01)[b], (192, 320))
        n = int(cnt[b])
        assert n == exp.shape[0] and n > 0 and torch.equal(out[b, :n, 5], exp[:, 5]) and torch.allclose(out[b, :n, :5], exp[:, :5], atol=1e-3)


def test_dropin_detector_modules_and_pipeline():
    """B-det boundary (attempt_load / model(img)[0] / non_max_suppression / scale_coords) and the 3-stream pipeline:
    the pipelined results equal the straight detect -> tracker sequence frame by frame."""
    import os, sys
    pkg = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "yolov7-tracker_b200")
    saved = {k: sys.modules.pop(k) for k in list(sys.modules) if k == "models" or k.startswith("models.") or k == "utils" or k.startswith("utils.")}
    sys.path.insert(0, pkg)
    g = torch.Generator().manual_seed(11)
    try:
        from models.experimental import attempt_load
        from utils.general import non_max_suppression, scale_coords, check_img_size
        from utils.torch_utils import select_device, time_synchronized
        from oracle import detector as OD
        device = select_device('0')
        model = attempt_load("seeded:0:256", map_location=device)
        assert int(model.stride.max()) == 64 and check_img_size(250, 64) == 256
        img = torch.rand((2, 3, 256, 256), generator=g)
        out = model(img.to(device))[0]
        assert tuple(out.shape) == (2, 4080, 85)
        dets = non_max_suppression(out, conf_thres=0.01)
        ref = OD.non_max_suppression(out, conf_thres=0.01)
        for a, b in zip(dets, ref):
            assert a.shape == b.shape and torch.equal(a[:, 5], b[:, 5]) and torch.allclose(a[:, :5], b[:, :5], atol=1e-3)
        d0 = dets[0].clone()
        d0[:, :4] = scale_coords((256, 256), d0[:, :4], (256, 256, 3), ratio_pad=None).round()        # tracker/track.py:240
        assert bool((d0[:, :4] >= 0).all()) and bool((d0[:, :4] <= 256).all())
        time_synchronized()
    finally:
        sys.path.remove(pkg)
        for k in list(sys.modules):
            if k == "models" or k.startswith("models.") or k == "utils" or k.startswith("utils."):
                sys.modules.pop(k)
        sys.modules.update(saved)
    # ---- pipeline == sequential
    from b200track.detector import DetectorW6
    from b200track.engine import TrackEngine
    from b200track.pipeline import TrackingPipeline
    from b200track.w6 import calibrated_state_dict
    from b200track import _lib as L
    sd = calibrated_state_dict(0, 256, "cuda")
    frames = [torch.roll(torch.rand((2, 3, 256, 256), generator=g), shifts=k, dims=3).pin_memory() for k in range(5)]
    det_a = DetectorW6(sd, batch=2, img_size=256, use_graph=False)
    eng_a = TrackEngine("bytetrack", n_seq=2, cap=512, dmax=300)
    seq = []
    for f in frames:
        det_a.detect(f.cuda(), post=True)
        t_out = torch.zeros((2, 512, L.OUT_COLS), dtype=torch.float64, device="cuda"); t_stat = torch.zeros((2, L.STAT_WORDS), dtype=torch.int32, device="cuda")
        eng_a.step_device(det_a.out, det_a.out_count, t_out, t_stat)
        torch.cuda.synchronize()
        seq.append([t_out[s, :int(t_stat[s, L.STAT_NOUT])].cpu().clone() for s in range(2)])
    det_b = DetectorW6(sd, batch=2, img_size=256, use_graph=False)
    eng_b = TrackEngine("bytetrack", n_seq=2, cap=512, dmax=300)
    pipe = TrackingPipeline(det_b, eng_b, out_rows=512)
    got = []
    for f in frames:
        r = pipe.step(f)
        if r is not None:
            got.append([r[0][s, :int(r[1][s, L.STAT_NOUT])].clone() for s in range(2)])
    r = pipe.flush()
    got.append([r[0][s, :int(r[1][s, L.STAT_NOUT])].clone() for s in range(2)])
    assert len(got) == len(seq)
    for a, b in zip(seq, got):
        for s in range(2):
            assert torch.equal(a[s], b[s])
