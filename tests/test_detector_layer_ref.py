"""not-gpu: the per-layer float64 harness (tests/detector_layer_ref.py) passes on a correct chain of stored layer outputs -- the
oracle's forward with the 16-bit rounding emulated -- and fails, at the right layer, on each kind of bug a detector kernel or its
buffer plan could have; its adapter maps every layer of a dry-run ``DetectorW6`` onto views of the oracle's shapes that do not overlap."""
import os
import sys

import pytest
import torch
import torch.nn.functional as F

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import detector_layer_ref as R  # noqa: E402
from plan_dryrun import dry_run_plan  # noqa: E402

DTYPES = [torch.float16, torch.bfloat16]


def _graph(name):
    from b200track import tiny, w6
    if name == "tiny320":                              # SP pools on a 10 x 10 map: the 9 and 13 windows differ
        return dict(_graph("tiny"), hw=(320, 320))
    if name == "w6":
        return dict(layers=w6.w6_layers(), sd=w6.calibrated_state_dict(0, 128, "cpu"), act="silu", anchors=w6.ANCHORS, strides=w6.STRIDES,
                    name_offset=0, hw=(128, 128))
    return dict(layers=tiny.tiny_layers(), sd=tiny.seeded_state_dict(0), act="leaky", anchors=tiny.ANCHORS, strides=tiny.STRIDES,
                name_offset=-1, hw=(128, 160))


_CHAINS = {}


def _chain(name, dtype):
    """(graph, image, store, pred) of the oracle at a small size, computed once per module."""
    if (name, dtype) not in _CHAINS:
        g = _graph(name)
        img = torch.rand((1, 3) + g["hw"], generator=torch.Generator().manual_seed(3))
        store, pred = R.oracle_chain(g["layers"], g["sd"], img, g["anchors"], g["strides"], dtype, act=g["act"], name_offset=g["name_offset"])
        _CHAINS[(name, dtype)] = (g, img, store, pred)
    return _CHAINS[(name, dtype)]


def _check(g, img, store, dtype, pred=None):
    return R.check_chain(g["layers"], g["sd"], g["act"], dtype, img, store.__getitem__, g["anchors"], g["strides"], name_offset=g["name_offset"], pred=pred)


@pytest.mark.parametrize("dtype", DTYPES, ids=["fp16", "bf16"])
@pytest.mark.parametrize("name", ["w6", "tiny"])
def test_harness_passes_on_correct_chain(name, dtype):
    g, img, store, pred = _chain(name, dtype)
    rows = _check(g, img, store, dtype, pred)
    print("\n" + R.format_table(rows, "%s %s %s" % (name, g["hw"], dtype)))
    assert not R.failures(rows), R.format_table(R.failures(rows))
    kinds = {r.kind for r in rows}
    assert kinds == {"exact", "conv", "head", "decode"}
    n_conv = sum(r.kind in ("conv", "head") for r in rows)
    assert n_conv == (107 if name == "w6" else 58)                     # every conv of the fused reference graph, stacked pairs split


# ---------------------------------------------------------------- mutations: each must fail, first at the layer it was made in

def _emulate_conv(x, w, b, k, s, act, dtype, rtz=False):
    """one conv as the kernel computes it (16-bit operands, fp32 sums), rounded to nearest or toward zero"""
    y = F.conv2d(x.float(), w.to(dtype).float(), b.float(), stride=s, padding=k // 2)
    y = y * torch.sigmoid(y) if act == "silu" else F.leaky_relu(y, 0.1)
    if not rtz:
        return y.to(dtype)
    y = y.double()
    q = R.ulp(y.abs(), dtype)
    return (torch.trunc(y / q) * q).to(dtype)


def _first_failure(name, dtype, mutate):
    g, img, store, pred = _chain(name, dtype)
    st = dict(store)
    mutate(g, st)
    bad = R.failures(_check(g, img, st, dtype))
    assert bad, "the mutation was not caught"
    return bad[0].key


def _conv_in(g, st, i):
    L = g["layers"]
    j = R._resolve(i, L[i][2])
    if L[j][1] == "concat":
        return torch.cat([st[R._resolve(j, f)] for f in L[j][2]], 1)
    return st[j]


def _recompute(g, st, i, dtype, w_edit=None, x_edit=None, rtz=False):
    L = g["layers"]
    _, op, frm, (cout, k, s) = L[i]
    nm = "model.%d.conv" % (i + g["name_offset"])
    w = g["sd"][nm + ".weight"].clone()
    x = _conv_in(g, st, i)
    if w_edit:
        w = w_edit(w)
    if x_edit:
        x = x_edit(x)
    st[i] = _emulate_conv(x, w, g["sd"][nm + ".bias"], k, s, g["act"], dtype, rtz)


def test_mutation_one_element_two_ulps_beyond_its_bound():
    dt = torch.float16

    def m(g, st):
        i = 20
        _, _, frm, (cout, k, s) = g["layers"][i]
        w = g["sd"]["model.%d.conv.weight" % i].to(dt).double()
        b = g["sd"]["model.%d.conv.bias" % i].double()
        ref, bound = R.conv_reference(_conv_in(g, st, i).double(), w, b, k, s, "silu", dt)
        e = (0, 5, 3, 4)
        v = ref[e] + bound[e] + 2 * R.ulp(ref[e].abs(), dt)
        t = st[i].clone()
        t[e] = R.round_nearest(v, dt).to(dt)
        st[i] = t
    assert _first_failure("w6", dt, m) == 20


def test_mutation_k_chunk_dropped_in_the_largest_k_layer():
    dt = torch.float16
    g = _chain("w6", dt)[0]
    convs = [(l[3][1] ** 2 * g["sd"]["model.%d.conv.weight" % l[0]].shape[1], l[0]) for l in g["layers"] if l[1] == "conv"]
    i = max(convs)[1]

    def drop(w):
        w[:, 128:192, 1, 1] = 0                        # one 64-channel chunk of one tap
        return w
    assert _first_failure("w6", dt, lambda g, st: _recompute(g, st, i, dt, w_edit=drop)) == i


def test_mutation_3x3_tap_dropped():
    dt = torch.float16

    def drop(w):
        w[:, :, 0, 2] = 0
        return w
    assert _first_failure("w6", dt, lambda g, st: _recompute(g, st, 5, dt, w_edit=drop)) == 5


def test_mutation_round_toward_zero_in_a_leaky_layer_of_tiny():
    dt = torch.float16
    assert _first_failure("tiny", dt, lambda g, st: _recompute(g, st, 2, dt, rtz=True)) == 2


def test_mutation_two_concat_slices_swapped():
    i = 9                                              # the first ELAN concat: [conv 8 | conv 6 | conv 4 | conv 3], 64 channels each

    def m(g, st):
        assert g["layers"][i][1] == "concat"
        t = st[i].clone()
        t[:, 0:64], t[:, 64:128] = st[i][:, 64:128], st[i][:, 0:64]
        st[i] = t
    assert _first_failure("w6", torch.float16, m) == i


def test_mutation_upsample_shifted_by_one_pixel():
    i = 49

    def m(g, st):
        assert g["layers"][i][1] == "up"
        st[i] = torch.roll(st[i], 1, dims=3)
    assert _first_failure("w6", torch.float16, m) == i


def test_mutation_spp_9_and_13_pools_swapped():
    """tiny at 320 x 320 (w6 at 128 x 128 pools a 2 x 2 map, where the two windows agree)"""
    g = _chain("tiny320", torch.float16)[0]
    i9, i13 = (next(l[0] for l in g["layers"] if l[1] == "sp" and l[3][0] == k) for k in (9, 13))

    def m(g, st):
        st[i9], st[i13] = st[i13], st[i9]
    assert _first_failure("tiny320", torch.float16, m) == i9


def test_mutation_rows_of_a_stacked_pair_swapped():
    from b200track.w6 import stackable_pairs
    i, j = stackable_pairs()[3]

    def m(g, st):
        st[i], st[j] = st[j], st[i]
    assert _first_failure("w6", torch.float16, m) == i


def test_mutation_tiny_sp_permutation_ignored():
    """the conv after tiny's SPP concat reads the buffer order [x | m5 | m9 | m13] with the reference's (unpermuted) weights"""
    dt = torch.float16
    g = _chain("tiny", dt)[0]
    ci = next(l[0] for l in g["layers"] if l[1] == "concat" and any(g["layers"][R._resolve(l[0], f)][1] == "sp" for f in l[2]))
    i = ci + 1

    def m(g, st):
        srcs = [R._resolve(ci, f) for f in g["layers"][ci][2]]          # reference order [m13, m9, m5, x]
        _recompute(g, st, i, dt, x_edit=lambda x: torch.cat([st[j] for j in srcs[::-1]], 1))
    assert _first_failure("tiny", dt, m) == i


def test_mutation_tile_left_at_sentinel():
    def m(g, st):
        t = st[10].clone()
        flat = t.permute(0, 2, 3, 1).reshape(-1, t.shape[1])                                   # pixels in NHWC order
        flat[128:256] = float("nan")
        st[10] = flat.view(t.shape[0], t.shape[2], t.shape[3], t.shape[1]).permute(0, 3, 1, 2)
    assert _first_failure("w6", torch.float16, m) == 10


def test_bound_catches_one_ulp_on_exact_pre_activation():
    """the bar is tight where the arithmetic is exact: a 1x1 identity conv (sum|w x| = |x|, E ~ 2^-21 |x|) must reject a one-ulp miss"""
    x = torch.tensor([1.0, -3.0, 0.01, 100.0], dtype=torch.float64).view(1, 4, 1, 1)
    w = torch.eye(4, dtype=torch.float64).view(4, 4, 1, 1)
    ref, bound = R.conv_reference(x, w, torch.zeros(4, dtype=torch.float64), 1, 1, "leaky", torch.float16)
    assert torch.equal(ref, torch.where(x >= 0, x, 0.1 * x))
    assert bool((R.ulp(ref.abs(), torch.float16) > bound).all())


def test_ulp_and_round_nearest_match_torch_casts():
    for dt in (torch.float16, torch.bfloat16):
        v = torch.cat([torch.randn(100000, dtype=torch.float64) * 10 ** torch.randint(-9, 4, (100000,)).double(), torch.tensor([0.0, 2.0 ** -30, 65504.0])])
        if dt == torch.float16:
            v = v.clamp(-65504, 65504)
        r = R.round_nearest(v, dt)
        assert torch.equal(r, v.float().to(dt).double()) or float((r != v.float().to(dt).double()).float().mean()) < 1e-4   # casts round twice
        assert torch.equal(r.to(dt).double(), r)                                                     # representable
        assert bool(((r - v).abs() <= 0.5 * R.ulp(v.abs(), dt)).all())


# ---------------------------------------------------------------- adapter wiring on dry-run detectors

def _meta_shapes(layers, act, anchors, strides, name_offset, B, H, W):
    from b200track.w6 import conv_shapes
    from oracle import detector as OD
    sd = {}
    for nm, cin, cout, k, s, _ in conv_shapes(layers, name_offset=name_offset):
        sd[nm + ".weight"] = torch.empty((cout, cin, k, k), device="meta")
        sd[nm + ".bias"] = torch.empty((cout,), device="meta")
    res = OD.forward(layers, sd, torch.empty((B, 3, H, W), device="meta"), anchors, strides, act=act, name_offset=name_offset, return_layers=True)
    shapes = {i: tuple(t.shape) for i, t in enumerate(res["layers"]) if t is not None}
    for i, d in res["spp"].items():
        shapes.update({("spp", i, nm): tuple(t.shape) for nm, t in d.items()})
    shapes.update({("raw", lvl): tuple(t.shape) for lvl, t in enumerate(res["raw"])})
    return shapes


@pytest.mark.parametrize("case", [("w6", 2, (256, 256)), ("w6", 1, (960, 1280)), ("tiny", 2, (192, 256))], ids=["w6-256", "w6-960x1280", "tiny-192x256"])
def test_adapter_views_have_oracle_shapes_and_do_not_overlap(case):
    from b200track import tiny, w6
    name, B, (H, W) = case
    det, _ = dry_run_plan(B, (H, W), tiny=name == "tiny")
    if name == "w6":
        layers, act, anchors, strides, no_ = w6.w6_layers(), "silu", w6.ANCHORS, w6.STRIDES, 0
    else:
        layers, act, anchors, strides, no_ = tiny.tiny_layers(), "leaky", tiny.ANCHORS, tiny.STRIDES, -1
    shapes = _meta_shapes(layers, act, anchors, strides, no_, B, H, W)
    views = R.detector_views(det, layers)
    assert set(views) == set(shapes)
    for key, v in views.items():
        want = shapes[key]
        if key == 0:                                   # the stem / input buffer carries 16 channels, the padding zeros
            want = (want[0], 16) + want[2:]
        assert tuple(v.shape) == want, (key, tuple(v.shape), want)
    # no two views overlap, except a concat with its own sources
    spans = R.detector_spans(det, layers)
    concat = {i: {R._resolve(i, f) for f in l[2]} for i, l in enumerate(layers) if l[1] == "concat"}
    keys = list(spans)
    for a in range(len(keys)):
        for b in range(a + 1, len(keys)):
            ka, kb = keys[a], keys[b]
            (ba, oa, ca), (bb, ob, cb) = spans[ka], spans[kb]
            if ba.data_ptr() != bb.data_ptr() or oa + ca <= ob or ob + cb <= oa:
                continue
            pair = {ka, kb}
            ok = any(ci in pair and (pair - {ci}) <= srcs for ci, srcs in concat.items())
            assert ok, "views %r and %r overlap" % (ka, kb)
    # every source lies inside its concat's buffer, at the channels the concat reads in reference order
    for ci, srcs in concat.items():
        assert all(spans[j][0] is spans[ci][0] for j in srcs)
