"""-m gpu: every conv plan the autotuner can pick, at every launch of real detector forwards, bit for bit against the plan the
detector ran; and the whole ConvPlan mode space against float64 (tests/conv_plan_ref.py).

Part a, every candidate at every launch.  For each configuration (the bench's w6 1280 x 1280 batch 8 fp16 autotuned; w6 768 x 1280
batch 2 bf16; w6 192 x 320 batch 2 fp16, maps down to 3 x 5; tiny 1280 x 1280 batch 1 fp16 autotuned) the layer buffers are filled
with NaN, frame A runs, then frame B, and the stored chain is checked against float64 (tests/detector_layer_ref.py).  Then, for every
launch (``DetectorW6.conv_specs``) and every candidate of ``conv_candidates`` -- the list the autotuner times -- a plan reads the
detector's real input buffer and writes into a NaN-filled clone of its destination buffer (often a concat buffer whose other slices
are this launch's inputs).  The launch's channel slice must equal the detector's stored slice bit for bit, every element outside the
slice (and its 16-byte store granule tail) must still be NaN, the input buffer must not change, and a second run into a refilled
clone must give the same bits.  A refused candidate must be refused by ``b2t_conv_plan_create``'s checks.  On a mismatch the
candidate is checked against float64 too, and the message says whether it is out of bound or only summed in another order.

Part b, the ConvPlan mode space.  The geometries of the torch-bar conv tests (test_gpu_detector.py, test_gpu_conv_schedule.py),
restated, plus a 3 x 5 map, a Cout of 40 and a 32-channel layer: BK 16 / 32 / 64, k 1 / 3, stride 1 / 2, ragged maps, flat tiles that
span two images, Cout not a multiple of 16 (the 255-channel fp32 head included), concat slices with pitch extras, the padded stem in
its three addressing modes; act 0 / 1 / 3, fp16 and bf16, 16-bit and fp32 output.  Covering rule, per geometry and addressing mode
(one tile per tap and halo; the stem's row-packed, nine-tap and halo): the default plan; every value of every knob on its own, the
others at their defaults -- block_n 32 / 64 / 128 / 256, mt 1 / 2, stages 0-4, producers 1 / 2, splits 1-4, out_bufs 1 / 2, and
tile_w 4 / 8 / 16 and kpair 1 / 2 (one tile per tap) or tps 1 / 3 / 9 and halo_bufs 2 / 3 (halo); and mt 2 with each BLOCK_N.
Every plan ``b2t_conv_plan_create`` accepts runs twice (bit-identical), is checked against the float64 bound with its own splits
term, and keeps the NaN around its slice; plans with one K split at a geometry give the same bits.  Every knob value is accepted at
some geometry (test_sweep_reaches_every_knob_value).
"""
import collections
import os
import sys
import time

import pytest

pytestmark = pytest.mark.gpu
torch = pytest.importorskip("torch")

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import conv_plan_ref as CR  # noqa: E402
import test_gpu_detector_layers as DL  # noqa: E402

NAN = float("nan")


def _bits(t):
    return t.view(torch.int32 if t.dtype == torch.float32 else torch.int16)


def _same_bits(a, b):
    return torch.equal(_bits(a), _bits(b))


def _refused_by_checks(e):
    """ConvPlan raises "b2t_conv_plan_create: <the library's message>"; a validation refusal's message names the function itself,
    a CUDA failure (tensor map encoding, allocation) does not"""
    return str(e).split(": ", 1)[-1].startswith("b2t_conv_plan_create:")


def _schedule(info, extra):
    return (info["pingpong"], info["mt"], info["bn"], info["stages"], info["kpair"], info["halo"], int(bool(extra.get("rowpack"))))


def _schedule_table(scheds):
    names = ("pingpong", "mt", "BLOCK_N", "stages", "kpair", "halo", "rowpack")
    return "  ".join("%s %s" % (n, sorted({s[i] for s in scheds})) for i, n in enumerate(names))


# ---------------------------------------------------------------- part a: every candidate at every launch

CONFIGS = [
    # id, graph, batch, (H, W), dtype, autotune / CUDA graph, images checked against float64 (None: all)
    ("w6-1280-b8-fp16-tuned", "w6", 8, (1280, 1280), torch.float16, True, (0, 7)),
    ("w6-768x1280-b2-bf16", "w6", 2, (768, 1280), torch.bfloat16, False, None),
    ("w6-192x320-b2-fp16", "w6", 2, (192, 320), torch.float16, False, None),
    ("tiny-1280-b1-fp16-tuned", "tiny", 1, (1280, 1280), torch.float16, True, None),
]


def _float64_verdict(det, sp, y):
    """for a mismatching candidate: 'out of bound' or 'within bound (summed in another order)'"""
    vi = next(i for i, (_, e) in enumerate(sp["variants"]) if not e.get("rowpack"))
    wpk, extra = sp["variants"][vi]
    k, cin, cout = sp["k"], sp["cin"], sp["cout"]
    x = CR.input_nchw(sp["src"], sp["in_coff"], cin, sp["hw_in"][1], extra.get("x_pixel0", 0))
    ref = CR.ConvRef(x, CR.unpack_weight(wpk, cout, cin, k), sp["bias"], k, sp["s"], sp["act"], det.act_dtype, sp["f32"])
    r, bnd = ref(1)
    c = CR.check_output(y, sp["out_coff"], cout, r, bnd, torch.float32 if sp["f32"] else det.act_dtype)
    return "err/bound %.3g: %s" % (c.max_ratio, "out of bound" if not c.ok else "within bound, summed in another order")


def _every_candidate(det, sp, stats):
    from b200track._lib import B2TError
    from b200track.conv import ConvPlan
    from b200track.detector import conv_candidates
    src, dst, oc, cout = sp["src"], sp["dst"], sp["out_coff"], sp["cout"]
    h, w = sp["hw_in"]
    stored = dst[..., oc:oc + cout]
    end = CR.granule_end(oc, cout, sp["f32"])
    src_before = src.clone()
    y = torch.empty_like(dst)
    problems = []
    cands = conv_candidates(sp["k"], sp["s"], sp["cin"], cout, sp["f32"], sp["variants"])
    for vi, cfg in cands:
        wpk, extra = sp["variants"][vi]
        y.fill_(NAN)
        try:
            plan = ConvPlan(src, wpk, sp["bias"], y, det.B, h, w, sp["cin"], sp["in_coff"], cout, sp["k"], sp["s"], oc, act=sp["act"],
                            out_f32=sp["f32"], **cfg, **extra)
        except B2TError as e:
            stats["refused"] += 1
            if not _refused_by_checks(e):
                problems.append("%s variant %d %s: not a validation refusal: %s" % (sp["name"], vi, cfg, e))
            continue
        stats["run"] += 1
        stats["sched"].add(_schedule(plan.info, extra))
        for attempt in ("first run", "second run"):
            if attempt == "second run":
                y.fill_(NAN)
            plan.run()
            torch.cuda.synchronize()
            what = []
            if not _same_bits(y[..., oc:oc + cout], stored):
                what.append("slice differs from the detector's (%s)" % _float64_verdict(det, sp, y))
            if not (bool(torch.isnan(y[..., :oc]).all()) and bool(torch.isnan(y[..., end:]).all())):
                what.append("wrote outside its slice")
            if what:
                problems.append("%s variant %d %s, %s: %s" % (sp["name"], vi, cfg, attempt, "; ".join(what)))
                break
        del plan
    if not _same_bits(src, src_before):
        problems.append("%s: an input buffer changed" % sp["name"])
    return problems


@pytest.mark.parametrize("cfg", CONFIGS, ids=[c[0] for c in CONFIGS])
def test_every_candidate_at_every_launch(cfg):
    from b200track.detector import conv_candidates
    cid, name, B, (H, W), dt, tuned, images = cfg
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    t0 = time.time()
    det = DL._make(name, B, (H, W), act_dtype=dt, autotune=tuned, use_graph=tuned)
    img = DL._run_a_then_b(det, B, H, W)
    rows = DL._check(name, det, img, images, "%s, frame B after A" % cid)
    worst = max((r for r in rows if r.kind in ("conv", "head")), key=lambda r: r.max_ratio)
    t1 = time.time()
    stats = dict(run=0, refused=0, sched=set())
    problems = []
    for sp in det.conv_specs:
        cands = conv_candidates(sp["k"], sp["s"], sp["cin"], sp["cout"], sp["f32"], sp["variants"])
        if tuned:
            if sp["chosen"] not in cands:
                problems.append("%s: the autotuner's choice %s is not an enumerated candidate" % (sp["name"], sp["chosen"]))
        elif sp["chosen"][1] != {}:
            problems.append("%s: the untuned detector runs %s, not the default tiling" % (sp["name"], sp["chosen"]))
        problems += _every_candidate(det, sp, stats)
    torch.cuda.synchronize()
    print("\n%s: %d launches, %d candidates run, %d refused; float64 chain check largest err/bound %.3g (%s); %.0f s build + chain, "
          "%.0f s candidates\n  schedules reached (%d): %s"
          % (cid, len(det.conv_specs), stats["run"], stats["refused"], worst.max_ratio, worst.name, t1 - t0, time.time() - t1,
             len(stats["sched"]), _schedule_table(stats["sched"])))
    del det
    torch.cuda.empty_cache()
    assert not problems, "%d problems:\n%s" % (len(problems), "\n".join(problems[:40]))


# ---------------------------------------------------------------- part b: the ConvPlan mode space against float64

GEOMETRIES = [
    # id, (n, h, w, cin, cout, k, s, in_pitch_extra, in_coff, out_pitch_extra, out_coff, act, f32)
    ("flat_64", (2, 32, 32, 64, 64, 1, 1, 0, 0, 0, 0, 1, False)),
    ("flat_span_images", (2, 24, 20, 256, 192, 1, 1, 0, 0, 0, 0, 1, False)),        # 480 pixels per image: tiles span two images
    ("flat_bn32", (2, 24, 24, 64, 32, 1, 1, 0, 0, 0, 0, 3, False)),
    ("flat_cout40_leaky", (1, 20, 20, 64, 40, 1, 1, 0, 0, 0, 0, 3, False)),         # Cout not a multiple of 16
    ("flat_long_k", (1, 40, 40, 1536, 384, 1, 1, 0, 0, 0, 0, 1, False)),
    ("flat_concat_slices", (2, 16, 16, 128, 64, 1, 1, 64, 64, 64, 32, 1, False)),
    ("flat_ragged_267", (1, 178, 192, 64, 64, 1, 1, 0, 0, 0, 0, 1, False)),
    ("head_20x20_f32", (2, 20, 20, 512, 255, 1, 1, 0, 0, 0, 0, 0, True)),
    ("head_3x5_f32", (2, 3, 5, 1024, 255, 1, 1, 0, 0, 0, 0, 0, True)),
    ("3x3_32x32", (2, 32, 32, 64, 64, 3, 1, 0, 0, 0, 0, 1, False)),
    ("3x3_concat_slices", (2, 40, 40, 128, 192, 3, 1, 64, 64, 128, 64, 1, False)),
    ("3x3_bk16", (1, 64, 64, 16, 64, 3, 1, 0, 0, 0, 0, 1, False)),
    ("3x3_bk16_36x24", (1, 36, 24, 16, 128, 3, 1, 0, 0, 0, 0, 3, False)),
    ("3x3_bk32", (2, 40, 56, 32, 64, 3, 1, 0, 0, 0, 0, 1, False)),
    ("3x3_20x20", (2, 20, 20, 256, 256, 3, 1, 0, 0, 0, 0, 1, False)),
    ("3x3_ragged_24x44", (1, 24, 44, 64, 64, 3, 1, 0, 0, 0, 0, 1, False)),
    ("3x3_3x5", (2, 3, 5, 512, 256, 3, 1, 0, 0, 0, 0, 1, False)),
    ("3x3_fp32_out", (2, 20, 20, 128, 96, 3, 1, 0, 0, 0, 0, 1, True)),
    ("s2_64x64", (1, 64, 64, 64, 128, 3, 2, 0, 0, 0, 0, 1, False)),
    ("s2_48x40", (2, 48, 40, 128, 192, 3, 2, 0, 0, 0, 0, 3, False)),
    ("s2_80x80_3n", (1, 80, 80, 512, 768, 3, 2, 0, 0, 0, 0, 1, False)),
    ("s2_6x10_to_3x5", (2, 6, 10, 256, 128, 3, 2, 0, 0, 0, 0, 1, False)),
    ("stem_padded", "stem"),
]

BASE_KNOBS = [("block_n", (32, 64, 128, 256)), ("mt", (1, 2)), ("stages", (0, 1, 2, 3, 4)), ("producers", (1, 2)), ("splits", (1, 2, 3, 4)),
              ("out_bufs", (1, 2))]
TAP_KNOBS = [("tile_w", (4, 8, 16)), ("kpair", (1, 2))]
HALO_KNOBS = [("tps", (1, 3, 9)), ("halo_bufs", (2, 3))]
ALL_KNOBS = BASE_KNOBS + TAP_KNOBS + HALO_KNOBS


def _sweep(addressing):
    """the covering set of plan arguments for one geometry (module docstring)"""
    out = []
    for a in addressing:
        knobs = BASE_KNOBS + (HALO_KNOBS if a.get("halo") else TAP_KNOBS)
        cands = [dict(a)] + [dict(a, **{kn: v}) for kn, vals in knobs for v in vals] + [dict(a, mt=2, block_n=bn) for bn in (32, 64, 128)]
        for c in cands:
            if c not in out:
                out.append(c)
    return out


def _setup(geo, dt):
    """-> (x, [(packed weights, addressing)], bias, y, plan geometry kwargs, ConvRef, out dtype)"""
    from b200track.conv import pack_conv_weight, pack_conv_weight_rowpack
    g = torch.Generator(device="cuda").manual_seed(sum(map(ord, geo[0])))
    if geo[1] == "stem":
        n, h, w, cout = 2, 48, 80, 64
        row = w + 8
        x = torch.zeros((n, h, row, 16), device="cuda", dtype=dt)
        x[:, :, 1:w + 1, :12] = torch.randn((n, h, w, 12), device="cuda", generator=g).to(dt)
        wt = torch.zeros((cout, 16, 3, 3), device="cuda")
        wt[:, :12] = torch.randn((cout, 12, 3, 3), device="cuda", generator=g) * (1.5 / 108 ** 0.5)
        b = torch.randn(cout, device="cuda", generator=g) * 0.5
        wp = pack_conv_weight(wt, dtype=dt)
        addressing = [(pack_conv_weight_rowpack(wt, dtype=dt), dict(rowpack=True, in_row_pixels=row, x_pixel0=0)),
                      (wp, dict(in_row_pixels=row, x_pixel0=1)), (wp, dict(in_row_pixels=row, x_pixel0=1, halo=True))]
        y = torch.full((n, h, w, cout), NAN, device="cuda", dtype=dt)
        kw = dict(n=n, h=h, w=w, cin=16, in_coff=0, cout=cout, k=3, stride=1, out_coff=0, act=1, out_f32=False)
        ref = CR.ConvRef(CR.input_nchw(x, 0, 16, w, 1), wt.to(dt), b, 3, 1, 1, dt, False)
        return x, addressing, b, y, kw, ref, dt
    n, h, w, cin, cout, k, s, ipx, icoff, opx, ocoff, act, f32 = geo[1]
    in_pitch = cin + ipx + (icoff if ipx == 0 else 0)
    x = torch.randn((n, h, w, in_pitch), device="cuda", generator=g).to(dt)
    wt = torch.randn((cout, cin, k, k), device="cuda", generator=g) * (1.5 / (cin * k * k) ** 0.5)
    b = torch.randn(cout, device="cuda", generator=g) * 0.5
    ho, wo = (h + 2 * (k // 2) - k) // s + 1, (w + 2 * (k // 2) - k) // s + 1
    out_dt = torch.float32 if f32 else dt
    y = torch.full((n, ho, wo, (cout + 7) // 8 * 8 + opx), NAN, device="cuda", dtype=out_dt)
    wp = pack_conv_weight(wt, dtype=dt)
    kw = dict(n=n, h=h, w=w, cin=cin, in_coff=icoff, cout=cout, k=k, stride=s, out_coff=ocoff, act=act, out_f32=f32)
    ref = CR.ConvRef(CR.input_nchw(x, icoff, cin, w), wt.to(dt), b, k, s, act, dt, f32)
    return x, [(wp, {}), (wp, dict(halo=True))], b, y, kw, ref, out_dt


def _plan(x, wpk, b, y, kw, args):
    from b200track.conv import ConvPlan
    return ConvPlan(x, wpk, b, y, kw["n"], kw["h"], kw["w"], kw["cin"], kw["in_coff"], kw["cout"], kw["k"], kw["stride"], kw["out_coff"],
                    act=kw["act"], out_f32=kw["out_f32"], **args)


def _plans(geo, dt):
    """every (plan arguments, ConvPlan or the refusal) of the sweep at one geometry"""
    from b200track._lib import B2TError
    x, addressing, b, y, kw, ref, out_dt = _setup(geo, dt)
    for wpk, a in addressing:
        for args in _sweep([a]):
            try:
                yield args, _plan(x, wpk, b, y, kw, args), (x, y, kw, ref, out_dt)
            except B2TError as e:
                yield args, e, (x, y, kw, ref, out_dt)


@pytest.mark.parametrize("dt", [torch.float16, torch.bfloat16], ids=["fp16", "bf16"])
@pytest.mark.parametrize("geo", GEOMETRIES, ids=[g[0] for g in GEOMETRIES])
def test_plan_modes_vs_float64(geo, dt):
    from b200track._lib import B2TError
    run, refused, worst, problems = 0, 0, 0.0, []
    one_split = None
    scheds = set()
    for args, plan, (x, y, kw, ref, out_dt) in _plans(geo, dt):
        if isinstance(plan, B2TError):
            refused += 1
            if not _refused_by_checks(plan):
                problems.append("%s: not a validation refusal: %s" % (args, plan))
            continue
        run += 1
        scheds.add(_schedule(plan.info, args))
        y.fill_(NAN)
        plan.run()
        torch.cuda.synchronize()
        first = y.clone()
        y.fill_(NAN)
        plan.run()
        torch.cuda.synchronize()
        if not _same_bits(first, y):
            problems.append("%s: a second run gives other bits" % args)
        r, bnd = ref(plan.info["splits"])
        c = CR.check_output(first, kw["out_coff"], kw["cout"], r, bnd, out_dt)
        worst = max(worst, c.max_ratio if c.nonfinite == 0 else float("inf"))
        if not c.ok:
            problems.append("%s (info %s): %s, max err/bound %.3g" % (args, {k: plan.info[k] for k in ("bn", "mt", "stages", "splits", "tps", "kpair")},
                                                                        c.where(), c.max_ratio))
        if plan.info["splits"] == 1:
            sl = first[..., kw["out_coff"]:kw["out_coff"] + kw["cout"]]
            if one_split is None:
                one_split = (args, sl)
            elif not _same_bits(sl, one_split[1]):
                problems.append("%s and %s (one K split each) give different bits" % (one_split[0], args))
        del plan
    print("\n%s %s: %d plans run, %d refused, largest err/bound %.3g, schedules %s" % (geo[0], dt, run, refused, worst, _schedule_table(scheds)))
    assert run > 0
    assert not problems, "%d problems:\n%s" % (len(problems), "\n".join(problems[:40]))


def test_sweep_reaches_every_knob_value():
    """each value of each knob is accepted by b2t_conv_plan_create at some geometry of the sweep (plans created, not run), and so are
    act 0 / 1 / 3, fp16 and bf16, 16-bit and fp32 output"""
    from b200track._lib import B2TError
    seen = collections.defaultdict(set)
    for dt in (torch.float16, torch.bfloat16):
        for geo in GEOMETRIES:
            for args, plan, (_, _, kw, _, out_dt) in _plans(geo, dt):
                if isinstance(plan, B2TError):
                    continue
                for kn, _ in ALL_KNOBS:
                    if kn in args:
                        seen[kn].add(args[kn])
                seen["halo"].add(int(bool(args.get("halo"))))
                seen["rowpack"].add(int(bool(args.get("rowpack"))))
                seen["act"].add(kw["act"])
                seen["dtype"].add(str(dt))
                seen["out"].add(str(out_dt))
                del plan
    missing = {kn: sorted(set(vals) - seen[kn]) for kn, vals in ALL_KNOBS if set(vals) - seen[kn]}
    print("\naccepted values: %s" % {k: sorted(v) for k, v in seen.items()})
    assert not missing, "knob values no geometry accepts: %s" % missing
    assert seen["act"] == {0, 1, 3} and seen["halo"] == {0, 1} and seen["rowpack"] == {0, 1} and len(seen["dtype"]) == 2
    assert seen["out"] == {"torch.float16", "torch.bfloat16", "torch.float32"}
