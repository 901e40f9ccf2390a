"""-m gpu: the conv kernel's pixel-run addressing (b2t_conv_desc.tile_w = 128: a sub-tile is 128 consecutive pixels of the flattened
N*Ho*Wo output axis, loaded per filter tap as one TMA im2col box) against float64 (tests/conv_plan_ref.py) and bit for bit against
the default spatial-patch plan of the same layer.

Geometries: the 20 x 20 and 40 x 40 maps of w6 at batch 8; runs that cross rows and images (2 x 24 x 20); ragged totals whose last
run passes the end of the tensor (2 x 3 x 5, 3 x 24 x 44); stride 2 into 20 x 20, into 3 x 5 and from an odd 7 x 9 map; concat
slices with pitch and channel offset on both sides; BK 64 / 32 / 16; act 0 / 1 / 3, fp16 and bf16, 16-bit and fp32 output.  At each,
the run plan with its defaults, every value of every knob on its own -- block_n 32 / 64 / 128 / 256, mt 1 / 2, stages 1-4, producers
1 / 2, splits 1-3, out_bufs 1 / 2 -- and mt 2 with each BLOCK_N.  Every plan ``b2t_conv_plan_create`` accepts runs twice with the
same bits, is within the float64 bound with its own splits term, keeps the NaN around its output slice, and gives the same bits as
the default spatial plan with the same K splits.  Every refusal is a validation refusal, and the layouts the mode does not cover
(1x1, halo, padded input rows) are refused.
"""
import os
import sys

import pytest

pytestmark = pytest.mark.gpu
torch = pytest.importorskip("torch")

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import conv_plan_ref as CR  # noqa: E402

NAN = float("nan")
RUNS = dict(tile_w=128)

GEOMETRIES = [
    # id, (n, h, w, cin, cout, k, s, in_pitch_extra, in_coff, out_pitch_extra, out_coff, act, f32)
    ("20x20_b8", (8, 20, 20, 256, 256, 3, 1, 0, 0, 0, 0, 1, False)),
    ("40x40_b8", (8, 40, 40, 128, 128, 3, 1, 0, 0, 0, 0, 1, False)),
    ("rows_and_images_2x24x20", (2, 24, 20, 64, 64, 3, 1, 0, 0, 0, 0, 1, False)),      # 480 pixels per image: runs cross both
    ("ragged_2x3x5", (2, 3, 5, 512, 256, 3, 1, 0, 0, 0, 0, 1, False)),                 # 30 pixels: the only run ends past the tensor
    ("ragged_3x24x44", (3, 24, 44, 64, 96, 3, 1, 0, 0, 0, 0, 3, False)),               # 3168 pixels = 24.75 runs
    ("s2_40x40_to_20x20", (4, 40, 40, 128, 192, 3, 2, 0, 0, 0, 0, 1, False)),
    ("s2_6x10_to_3x5", (2, 6, 10, 256, 128, 3, 2, 0, 0, 0, 0, 1, False)),
    ("s2_7x9_to_4x5", (3, 7, 9, 64, 64, 3, 2, 0, 0, 0, 0, 1, False)),                   # odd input: the last column / row has no right tap
    ("concat_slices", (2, 20, 20, 128, 192, 3, 1, 64, 64, 128, 64, 1, False)),
    ("bk32", (2, 20, 20, 32, 64, 3, 1, 0, 0, 0, 0, 1, False)),
    ("bk16", (1, 36, 24, 16, 128, 3, 1, 0, 0, 0, 0, 3, False)),
    ("fp32_out", (2, 20, 20, 128, 96, 3, 1, 0, 0, 0, 0, 0, True)),
]

KNOBS = [("block_n", (32, 64, 128, 256)), ("mt", (1, 2)), ("stages", (1, 2, 3, 4)), ("producers", (1, 2)), ("splits", (1, 2, 3)),
         ("out_bufs", (1, 2))]


def _bits(t):
    return t.view(torch.int32 if t.dtype == torch.float32 else torch.int16)


def _same_bits(a, b):
    return torch.equal(_bits(a), _bits(b))


def _refused_by_checks(e):
    """ConvPlan raises "b2t_conv_plan_create: <the library's message>"; a validation refusal's message names the function itself"""
    return str(e).split(": ", 1)[-1].startswith("b2t_conv_plan_create:")


def _sweep():
    out = [dict(RUNS)] + [dict(RUNS, **{kn: v}) for kn, vals in KNOBS for v in vals] + [dict(RUNS, mt=2, block_n=bn) for bn in (32, 64, 128)]
    return [c for i, c in enumerate(out) if c not in out[:i]]


def _setup(geo, dt):
    """-> (x, packed weights, bias, y, plan geometry kwargs, ConvRef, out dtype)"""
    from b200track.conv import pack_conv_weight
    g = torch.Generator(device="cuda").manual_seed(sum(map(ord, geo[0])))
    n, h, w, cin, cout, k, s, ipx, icoff, opx, ocoff, act, f32 = geo[1]
    in_pitch = cin + ipx + (icoff if ipx == 0 else 0)
    x = torch.randn((n, h, w, in_pitch), device="cuda", generator=g).to(dt)
    wt = torch.randn((cout, cin, k, k), device="cuda", generator=g) * (1.5 / (cin * k * k) ** 0.5)
    b = torch.randn(cout, device="cuda", generator=g) * 0.5
    ho, wo = (h + 2 * (k // 2) - k) // s + 1, (w + 2 * (k // 2) - k) // s + 1
    out_dt = torch.float32 if f32 else dt
    y = torch.full((n, ho, wo, (cout + 7) // 8 * 8 + opx), NAN, device="cuda", dtype=out_dt)
    kw = dict(n=n, h=h, w=w, cin=cin, in_coff=icoff, cout=cout, k=k, stride=s, out_coff=ocoff, act=act, out_f32=f32)
    ref = CR.ConvRef(CR.input_nchw(x, icoff, cin, w), wt.to(dt), b, k, s, act, dt, f32)
    return x, pack_conv_weight(wt, dtype=dt), b, y, kw, ref, out_dt


def _plan(x, wpk, b, y, kw, **args):
    from b200track.conv import ConvPlan
    return ConvPlan(x, wpk, b, y, kw["n"], kw["h"], kw["w"], kw["cin"], kw["in_coff"], kw["cout"], kw["k"], kw["stride"], kw["out_coff"],
                    act=kw["act"], out_f32=kw["out_f32"], **args)


def _run(plan, y):
    y.fill_(NAN)
    plan.run()
    torch.cuda.synchronize()
    return y.clone()


@pytest.mark.parametrize("dt", [torch.float16, torch.bfloat16], ids=["fp16", "bf16"])
@pytest.mark.parametrize("geo", GEOMETRIES, ids=[g[0] for g in GEOMETRIES])
def test_pixel_runs_vs_float64_and_spatial_plan(geo, dt):
    from b200track._lib import B2TError
    x, wpk, b, y, kw, ref, out_dt = _setup(geo, dt)
    oc, cout = kw["out_coff"], kw["cout"]
    spatial = {}                                  # K splits -> the default spatial plan's output slice

    def spatial_slice(splits):
        if splits not in spatial:
            p = _plan(x, wpk, b, y, kw, splits=splits)
            spatial[splits] = _run(p, y)[..., oc:oc + cout]
            del p
        return spatial[splits]

    run, refused, worst, problems, tiles = 0, 0, 0.0, [], set()
    for args in _sweep():
        try:
            plan = _plan(x, wpk, b, y, kw, **args)
        except B2TError as e:
            refused += 1
            if not _refused_by_checks(e):
                problems.append("%s: not a validation refusal: %s" % (args, e))
            continue
        run += 1
        info = plan.info
        tiles.add((info["mt"], info["bn"], info["tiles_m"]))
        first = _run(plan, y)
        if not _same_bits(first, _run(plan, y)):
            problems.append("%s: a second run gives other bits" % args)
        r, bnd = ref(info["splits"])
        c = CR.check_output(first, oc, cout, r, bnd, out_dt)
        worst = max(worst, c.max_ratio if c.nonfinite == 0 else float("inf"))
        if not c.ok:
            problems.append("%s (bn %d mt %d stages %d splits %d): %s, max err/bound %.3g" % (args, info["bn"], info["mt"], info["stages"],
                                                                                           info["splits"], c.where(), c.max_ratio))
        if not _same_bits(first[..., oc:oc + cout], spatial_slice(info["splits"])):
            problems.append("%s: bits differ from the spatial plan with %d K split(s)" % (args, info["splits"]))
        del plan
    n, ho, wo = kw["n"], y.shape[1], y.shape[2]
    print("\n%s %s: %d x %d x %d = %d output pixels; %d run plans, %d refused, largest err/bound %.3g; (mt, BLOCK_N, M tiles) %s"
          % (geo[0], dt, n, ho, wo, n * ho * wo, run, refused, worst, sorted(tiles)))
    assert run > 0
    # the M tiles are whole 128 * mt runs of the flattened output axis
    assert all(tm == -(-n * ho * wo // (128 * mt)) for mt, _, tm in tiles)
    assert not problems, "%d problems:\n%s" % (len(problems), "\n".join(problems[:40]))


def test_pixel_runs_refuse_what_they_do_not_cover():
    """1x1 layers (flat already), halo mode and padded input rows (the stem buffer) are refused, by validation"""
    from b200track._lib import B2TError
    from b200track.conv import pack_conv_weight
    dt = torch.float16
    n, h, w = 2, 20, 20
    cases = []
    x = torch.randn((n, h, w, 64), device="cuda").to(dt)
    y = torch.full((n, h, w, 64), NAN, device="cuda", dtype=dt)
    b = torch.zeros(64, device="cuda")
    w1 = pack_conv_weight(torch.randn((64, 64, 1, 1), device="cuda") * 0.1, dtype=dt)
    w3 = pack_conv_weight(torch.randn((64, 64, 3, 3), device="cuda") * 0.05, dtype=dt)
    kw = dict(n=n, h=h, w=w, cin=64, in_coff=0, cout=64, stride=1, out_coff=0, act=1, out_f32=False)
    cases.append(("1x1", x, w1, dict(kw, k=1), {}))
    cases.append(("halo", x, w3, dict(kw, k=3), dict(halo=True)))
    xr = torch.randn((n, h, w + 8, 64), device="cuda").to(dt)
    cases.append(("padded rows", xr, w3, dict(kw, k=3), dict(in_row_pixels=w + 8, x_pixel0=1)))
    problems = []
    for name, xx, wpk, g, extra in cases:
        try:
            plan = _plan(xx, wpk, b, y, g, **RUNS, **extra)
            problems.append("%s: accepted" % name)
            del plan
        except B2TError as e:
            if not _refused_by_checks(e):
                problems.append("%s: not a validation refusal: %s" % (name, e))
    assert not problems, "\n".join(problems)
