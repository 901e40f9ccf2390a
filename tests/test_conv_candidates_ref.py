"""not-gpu: the conv autotuner's candidate list (``b200track.detector.conv_candidates``) on dry-run plans, and the NHWC float64 checker
of tests/conv_plan_ref.py against bugs a conv kernel could have.

Candidates: every launch of the w6 (1280 x 1280, batch 8) and tiny plans is offered a non-empty list that holds the kernel's default
plan; the padded w6 stem offers its three addressing variants (row-packed, nine taps, halo), and the halo variant is offered exactly
where the layer is 3x3, stride 1, Cin a multiple of 64.

Checker: each injected bug must fail, at the place it was made, and the correctly rounded result must pass.  The first two bugs
(split-K partials stored in the 16-bit type, the accumulator rounded to 16 bits before the bias add) pass the torch fp32 bar the
older conv tests use (2e-3 + 2e-3 |ref| fp16, 1.5e-2 + 1.5e-2 |ref| bf16): that is why the conv tests compare with float64 instead.
"""
import os
import sys

import pytest
import torch
import torch.nn.functional as F

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import conv_plan_ref as CR  # noqa: E402
import detector_layer_ref as R  # noqa: E402
from plan_dryrun import dry_run_plan  # noqa: E402

DTYPES = [torch.float16, torch.bfloat16]
TORCH_TOL = {torch.float16: 2e-3, torch.bfloat16: 1.5e-2}
NAN = float("nan")


# ---------------------------------------------------------------- candidate lists on dry-run plans

def _default_bn(cout):
    """b2t_conv_plan_create's BLOCK_N when the caller does not choose: Cout padded to 16 up to 64, then 128 or 64, rounded up to an
    instantiated width (32, 64, 128, 256)"""
    cp = (cout + 15) // 16 * 16
    bn = cp if cp <= 64 else (128 if cp % 128 == 0 else 64)
    b = 32
    while b < bn:
        b *= 2
    return b


@pytest.mark.parametrize("case", [("w6", 8, 1280), ("tiny", 1, 1280)], ids=["w6-1280-b8", "tiny-1280-b1"])
def test_every_launch_is_offered_its_default_plan(case):
    from b200track.detector import conv_candidates
    name, B, S = case
    det, plan = dry_run_plan(B, S, tiny=name == "tiny")
    specs = det.conv_specs
    assert len(specs) == len(plan) == (96 if name == "w6" else 50)
    n_cand = 0
    for i, sp in enumerate(specs):
        k, s, cin, cout = sp["k"], sp["s"], sp["cin"], sp["cout"]
        extras = [e for _, e in sp["variants"]]
        cands = conv_candidates(k, s, cin, cout, sp["f32"], sp["variants"])
        n_cand += len(cands)
        assert cands, "launch %d (%s) has no candidate" % (i, sp["name"])
        assert all(0 <= vi < len(sp["variants"]) for vi, _ in cands)
        stem = i == 0 and det.stem_padded
        if stem:
            assert [(e.get("rowpack", False), e.get("x_pixel0"), e.get("halo", 0)) for e in extras] == [(True, 0, 0), (False, 1, 0), (False, 1, 1)]
            assert all(e["in_row_pixels"] == det.stem_row for e in extras)
        else:
            want_halo = k == 3 and s == 1 and cin % 64 == 0
            assert [bool(e.get("halo")) for e in extras] == ([False, True] if want_halo else [False]), (i, sp["name"])
        # the untuned detector runs the first variant with the kernel's default tiling: the autotuner must time it too
        assert sp["chosen"] == (0, {})
        kp = 2 if (k == 1 and s == 1 and cin % 128 == 0) else 0
        default = dict(block_n=_default_bn(cout), mt=1, stages=0, kpair=kp)
        assert (0, default) in cands, "launch %d (%s): default plan %s not offered" % (i, sp["name"], default)
        # the record points at the buffers the plan reads and writes
        x, w, b, y = det.keep[[j for j, p in enumerate(det.keep) if hasattr(p, "geom")][i]].keep
        assert x is sp["src"] and y is sp["dst"] and b is sp["bias"] and w is sp["variants"][0][0]
        assert plan[i]["in_coff"] == sp["in_coff"] and plan[i]["out_coff"] == sp["out_coff"] and plan[i]["cout"] == cout
    print("\n%s: %d launches, %d candidates" % (name, len(specs), n_cand))


def test_head_candidates_respect_the_fp32_accumulator_limit():
    """fp32 heads: mt = 2 only with BLOCK_N 64; 1x1 layers of whole 128-channel pairs get kpair 1 and 2, others the default"""
    from b200track.detector import conv_candidates
    c = conv_candidates(1, 1, 512, 255, True, [None])
    assert all(cfg["block_n"] == 64 for _, cfg in c if cfg["mt"] == 2)
    assert {cfg["kpair"] for _, cfg in c} == {1, 2}
    assert {cfg["kpair"] for _, cfg in conv_candidates(3, 1, 512, 256, False, [None, None])} == {0}
    assert {cfg["block_n"] for _, cfg in conv_candidates(1, 1, 64, 32, False, [None])} == {32, 64}


# ---------------------------------------------------------------- the checker against injected bugs

def _operands(n, h, w, cin, cout, k, dt, seed):
    """the operand statistics of the conv tests: x ~ N(0, 1) in the 16-bit type, w ~ N(0, 1.5^2 / (cin k^2)), bias ~ N(0, 0.25)"""
    g = torch.Generator().manual_seed(seed)
    x = torch.randn((n, cin, h, w), generator=g, dtype=torch.float64).to(dt).double()
    wt = (torch.randn((cout, cin, k, k), generator=g) * (1.5 / (cin * k * k) ** 0.5)).to(dt).double()
    b = (torch.randn(cout, generator=g) * 0.5).double()
    return x, wt, b


def _silu(v):
    return v * torch.sigmoid(v)


def _nhwc(t, dt, pitch=None, coff=0):
    """NCHW values -> an NHWC buffer of `pitch` channels filled with NaN, the values at channels [coff, coff + C)"""
    n, c, h, w = t.shape
    y = torch.full((n, h, w, pitch or c), NAN, dtype=dt)
    y[..., coff:coff + c] = t.permute(0, 2, 3, 1).to(dt)
    return y


def _check(y, ref, out_dtype, coff=0):
    r, bnd = ref
    return CR.check_output(y, coff, r.shape[1], r, bnd, out_dtype)


def _torch_bar_passes(y, x, wt, b, act, dt, coff=0):
    cout = wt.shape[0]
    r = F.conv2d(x.float(), wt.float(), b.float(), padding=wt.shape[-1] // 2)
    r = _silu(r) if act == "silu" else r
    got = y[..., coff:coff + cout].permute(0, 3, 1, 2).float()
    return bool(((got - r).abs() <= TORCH_TOL[dt] + TORCH_TOL[dt] * r.abs()).all())


@pytest.fixture(scope="module")
def long_k():
    """the 1x1 layer of the table: 40 x 40, Cin 1536 -> 384, SiLU, 3 K splits of 512 channels"""
    out = {}
    for dt in DTYPES:
        x, wt, b = _operands(1, 40, 40, 1536, 384, 1, dt, 1536)
        ref = CR.ConvRef(x, wt, b, 1, 1, 1, dt, False)
        parts = [F.conv2d(x[:, j:j + 512], wt[:, j:j + 512]) for j in range(0, 1536, 512)]
        out[dt] = (x, wt, b, ref, parts)
    return out


@pytest.mark.parametrize("dt", DTYPES, ids=["fp16", "bf16"])
def test_correctly_rounded_result_passes(long_k, dt):
    x, wt, b, ref, _ = long_k[dt]
    r, _ = ref(3)
    c = _check(_nhwc(R.round_nearest(r, dt), dt), ref(3), dt)
    assert c.ok and c.n_exact == c.n, c.where()


@pytest.mark.parametrize("dt", DTYPES, ids=["fp16", "bf16"])
def test_split_k_partials_stored_in_16_bits_fail(long_k, dt):
    x, wt, b, ref, parts = long_k[dt]
    acc = sum(R.round_nearest(p, dt) for p in parts)
    y = _nhwc(R.round_nearest(_silu(acc + b.view(1, -1, 1, 1)), dt), dt)
    c = _check(y, ref(3), dt)
    print("\nsplit-K partials in %s: %d elements over the float64 bound, max err/bound %.2f" % (dt, int(c.over.sum()), c.max_ratio))
    assert not c.ok and c.nonfinite == 0 and c.max_ratio > 1.0
    assert _torch_bar_passes(y, x, wt, b, "silu", dt), "the torch bar was expected to miss this bug"


@pytest.mark.parametrize("dt", DTYPES, ids=["fp16", "bf16"])
def test_accumulator_rounded_before_bias_fails(long_k, dt):
    x, wt, b, ref, parts = long_k[dt]
    acc = R.round_nearest(sum(parts), dt)
    y = _nhwc(R.round_nearest(_silu(acc + b.view(1, -1, 1, 1)), dt), dt)
    c = _check(y, ref(3), dt)
    print("\naccumulator rounded to %s before the bias: %d elements over the float64 bound, max err/bound %.2f" % (dt, int(c.over.sum()), c.max_ratio))
    assert not c.ok and c.max_ratio > 1.0
    assert _torch_bar_passes(y, x, wt, b, "silu", dt), "the torch bar was expected to miss this bug"


@pytest.mark.parametrize("dt", DTYPES, ids=["fp16", "bf16"])
def test_tap_dropped_on_the_last_tile_column_fails_there(dt):
    """3x3 on a 20 x 20 map: tiles of 4 x 32 pixels (20 is not a multiple of 8), the last tile column is x in [16, 20); the tap
    (kh 1, kw 0) is dropped for those pixels only"""
    x, wt, b = _operands(2, 20, 20, 64, 64, 3, dt, 3)
    ref = CR.ConvRef(x, wt, b, 3, 1, 1, dt, False)
    r, _ = ref()
    w2 = wt.clone()
    w2[:, :, 1, 0] = 0
    bad = _silu(F.conv2d(x, w2, padding=1) + b.view(1, -1, 1, 1))
    v = r.clone()
    v[..., 16:] = bad[..., 16:]
    c = _check(_nhwc(R.round_nearest(v, dt), dt), ref(), dt)
    assert not c.ok and c.nonfinite == 0
    cols = c.over.nonzero()[:, 3]
    assert bool((cols >= 16).all()), "failures outside the last tile column: %s" % sorted(set(cols.tolist()))


@pytest.mark.parametrize("dt", DTYPES, ids=["fp16", "bf16"])
def test_neighbouring_n_tile_bias_fails_in_that_tile(dt):
    """Cout 384 in BLOCK_N 128 tiles: tile 1 (channels 128-255) adds the bias of tile 2"""
    x, wt, b = _operands(1, 16, 16, 256, 384, 1, dt, 4)
    ref = CR.ConvRef(x, wt, b, 1, 1, 1, dt, False)
    b2 = b.clone()
    b2[128:256] = b[256:384]
    v = _silu(F.conv2d(x, wt) + b2.view(1, -1, 1, 1))
    c = _check(_nhwc(R.round_nearest(v, dt), dt), ref(), dt)
    assert not c.ok
    ch = c.over.nonzero()[:, 1]
    assert bool(((ch >= 128) & (ch < 256)).all()) and int(c.over[:, 128:256].sum()) > 0.9 * c.over[:, 128:256].numel()


def test_tile_left_at_the_sentinel_fails_there():
    """a 128-pixel x 64-channel tile of a flat layer never stored: exactly its elements are reported, as not finite"""
    dt = torch.float16
    x, wt, b = _operands(1, 16, 24, 64, 128, 1, dt, 5)
    ref = CR.ConvRef(x, wt, b, 1, 1, 1, dt, False)
    r, _ = ref()
    y = _nhwc(R.round_nearest(r, dt), dt)
    y.view(-1, 128)[128:256, 64:128] = NAN                              # pixels 128-255 in NHWC order, N tile 1
    c = _check(y, ref(), dt)
    assert not c.ok and c.nonfinite == 128 * 64
    over = c.over.permute(0, 2, 3, 1).reshape(-1, 128)
    assert bool(over[128:256, 64:128].all()) and int(over.sum()) == 128 * 64


@pytest.mark.parametrize("f32", [False, True], ids=["16-bit", "fp32"])
def test_write_one_granule_past_the_slice_fails_there(f32):
    """output slice [64, 64 + 196) of a 320-channel concat buffer, linear: the store granule tail (16-bit: channels 260-263, up to the
    next 16 bytes) may be written, the next granule may not, nor the channels just before the slice"""
    dt = torch.float16
    out_dt = torch.float32 if f32 else dt
    x, wt, b = _operands(1, 8, 8, 64, 196, 1, dt, 6)
    ref = CR.ConvRef(x, wt, b, 1, 1, 0, dt, f32)
    r, bnd = ref()
    y = _nhwc(R.round_nearest(r, out_dt), out_dt, pitch=320, coff=64)
    end = CR.granule_end(64, 196, f32)
    assert end == (260 if f32 else 264)
    y[..., 260:end] = 0.0                                                   # the granule tail the store owns
    c = CR.check_output(y, 64, 196, r, bnd, out_dt)
    assert c.ok, c.where()
    past = list(range(end, end + (4 if f32 else 8)))
    y[..., past] = 0.0                                                      # one granule past the slice
    c = CR.check_output(y, 64, 196, r, bnd, out_dt)
    assert not c.ok and c.max_ratio <= 1.0 and c.nonfinite == 0
    assert set(c.outside.nonzero()[:, 3].tolist()) == set(past)
    y[..., 60:64] = 0.0                                                     # and just before the slice
    assert set(CR.check_output(y, 64, 196, r, bnd, out_dt).outside.nonzero()[:, 3].tolist()) == set(past) | {60, 61, 62, 63}
