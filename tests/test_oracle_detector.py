"""not-gpu: the torch oracle of the detector against the committed outputs of the reference's own Model
(tests/golden/detector_w6.npz) -- pins both oracle/detector.py and the product's graph builder (w6_layers)."""
import os

import numpy as np
import pytest
import torch

from b200track.w6 import ANCHORS, STRIDES, conv_shapes, layer_channels, seeded_state_dict, w6_layers
from oracle import detector as OD

GOLDEN = os.path.join(os.path.dirname(__file__), "golden", "detector_w6.npz")
REFCHECKS = os.path.join(os.path.dirname(__file__), "golden", "refchecks.npz")


def test_graph_bookkeeping():
    layers = w6_layers()
    assert len(layers) == 119 and layers[-1][1] == "detect"
    ch = layer_channels(layers)
    assert ch[46] == 1024 and ch[47] == 512 and ch[83] == 128 and ch[117] == 1024 and ch[9] == 256 and ch[58] == 1536
    shapes = conv_shapes(layers)
    assert len(shapes) == 107                                    # SURVEY 8(a): 107 convs after fusion
    n_params = sum(ci * co * k * k + co for _, ci, co, k, s, _ in shapes)
    assert abs(n_params - 70.43e6) / 70.43e6 < 0.01              # 70.4 M parameters (SURVEY 8a)


def test_stackable_1x1_pairs_and_rowpack_layout():
    """Host logic of the detector planner: the 11 ELAN blocks each open with two 1x1 convs of the same input that are adjacent
    in the block's concat; the row-packed stem weight layout is k = kh*64 + kw*16 + c with a zero fourth pixel."""
    from b200track.w6 import stackable_pairs
    pairs = stackable_pairs()
    assert len(pairs) == 11 and pairs[0] == (3, 4) and (12, 13) in pairs and (50 + 2, 50 + 3) in pairs
    layers = w6_layers()
    for a, b in pairs:
        assert layers[a][1] == layers[b][1] == "conv" and layers[a][3] == layers[b][3] and layers[b][2] == -2
    from b200track.conv import pack_conv_weight_rowpack
    w = torch.arange(64 * 12 * 9, dtype=torch.float32).reshape(64, 12, 3, 3) / 4096.0
    pk = pack_conv_weight_rowpack(w).float().reshape(64, 3, 4, 16)
    assert torch.equal(pk[:, :, :3, :12], w.to(torch.bfloat16).float().permute(0, 2, 3, 1))
    assert bool((pk[:, :, 3] == 0).all()) and bool((pk[:, :, :, 12:] == 0).all())


def test_oracle_forward_and_nms_match_reference_golden():
    torch.set_num_threads(max(1, os.cpu_count() or 1))
    g = np.load(GOLDEN)
    sd = seeded_state_dict(0)
    gen = torch.Generator().manual_seed(123)
    img = torch.rand((1, 3, 256, 256), generator=gen)
    with torch.no_grad():
        pred = OD.forward(w6_layers(), sd, img, ANCHORS, STRIDES)
    assert tuple(pred.shape) == tuple(g["pred_shape"])
    np.testing.assert_allclose(pred[0, g["rows"]].numpy(), g["pred_rows"], rtol=2e-3, atol=2e-3)
    assert int((pred[0, :, 4] > 0.01).sum()) == int(g["n_candidates"])
    dets = OD.non_max_suppression(pred, conf_thres=0.01)[0].numpy()
    ref = g["dets"]
    assert dets.shape == ref.shape
    assert np.array_equal(dets[:, 5], ref[:, 5])                 # classes and order: exact
    np.testing.assert_allclose(dets[:, :5], ref[:, :5], rtol=2e-3, atol=2e-2)


def test_fold_batchnorm_and_implicit_layers_math():
    """fold_reference_state_dict on a synthetic one-layer problem: Conv + BN(eval) and ia / m / im head == the folded convs."""
    import torch.nn.functional as F
    from b200track.w6 import conv_shapes, fold_reference_state_dict
    g = torch.Generator().manual_seed(1)
    sd = {}
    for name, cin, cout, k, s, act in conv_shapes():
        if act:
            sd[name + ".weight"] = torch.randn((cout, cin, k, k), generator=g) * 0.05
            pre = name[:-len(".conv")]
            sd[pre + ".bn.weight"] = torch.rand(cout, generator=g) + 0.5
            sd[pre + ".bn.bias"] = torch.randn(cout, generator=g) * 0.1
            sd[pre + ".bn.running_mean"] = torch.randn(cout, generator=g) * 0.1
            sd[pre + ".bn.running_var"] = torch.rand(cout, generator=g) + 0.2
        else:
            j = int(name.rsplit(".", 1)[1])
            sd["model.122.m.%d.weight" % j] = torch.randn((cout, cin, 1, 1), generator=g) * 0.05
            sd["model.122.m.%d.bias" % j] = torch.randn(cout, generator=g) * 0.1
            sd["model.122.m2.%d.weight" % j] = torch.zeros((cout, 8, 1, 1))
            sd["model.122.ia.%d.implicit" % j] = torch.randn((1, cin, 1, 1), generator=g) * 0.02
            sd["model.122.im.%d.implicit" % j] = 1 + torch.randn((1, cout, 1, 1), generator=g) * 0.02
    out = fold_reference_state_dict(sd)
    assert set(out) == {n + s for n, *_ in conv_shapes() for s in (".weight", ".bias")}
    name = "model.5.conv"                                             # a 3x3 Conv + BN
    x = torch.randn((1, 64, 9, 9), generator=g)
    pre = "model.5"
    ref = F.batch_norm(F.conv2d(x, sd[name + ".weight"], None, padding=1), sd[pre + ".bn.running_mean"], sd[pre + ".bn.running_var"],
                       sd[pre + ".bn.weight"], sd[pre + ".bn.bias"], False, 0.03, 1e-3)
    got = F.conv2d(x, out[name + ".weight"], out[name + ".bias"], padding=1)
    assert torch.allclose(got, ref, atol=1e-5)
    x = torch.randn((1, 256, 5, 5), generator=g)                      # head 0: m(ia + x) * im
    ref = F.conv2d(x + sd["model.122.ia.0.implicit"], sd["model.122.m.0.weight"], sd["model.122.m.0.bias"]) * sd["model.122.im.0.implicit"]
    got = F.conv2d(x, out["model.118.m.0.weight"], out["model.118.m.0.bias"])
    assert torch.allclose(got, ref, atol=1e-5)
    assert fold_reference_state_dict(out).keys() == out.keys()        # an already fused dict passes through


def test_fold_training_checkpoint_equals_reference_inference():
    """The reference's own TRAINING graph (cfg/training/yolov7-w6.yaml: Conv + BN, aux heads, IAuxDetect with implicit layers) on a
    seeded state dict with randomised BN statistics, evaluated by the reference in eval mode (every objectness and a seeded sample of
    rows, tests/golden/refchecks.npz) == the oracle forward on the folded deploy-graph weights.  The state dict is regenerated here
    from the same seed over the reference's key names and shapes, which the archive stores."""
    from b200track.w6 import fold_reference_state_dict
    g = np.load(REFCHECKS)
    keys = [str(k) for k in g["fold_keys"]]
    shapes = [[v for v in row if v >= 0] for row in g["fold_shapes"]]
    sd = OD.seeded_training_state_dict(keys, shapes, 3)
    img = torch.rand((1, 3, 128, 128), generator=torch.Generator().manual_seed(4))
    folded = fold_reference_state_dict(sd)
    with torch.no_grad():
        got = OD.forward(w6_layers(), folded, img, ANCHORS, STRIDES).double().numpy()
    assert got.shape == tuple(g["fold_shape"])
    rows = got.reshape(-1, got.shape[-1])[g["fold_row_index"]]
    np.testing.assert_allclose(rows, g["fold_rows"], rtol=2e-3, atol=2e-3)
    np.testing.assert_allclose(got[..., 4], g["fold_obj"], rtol=2e-3, atol=2e-3)


def test_tiny_oracle_equals_reference_model():
    """YOLOv7-tiny (cfg/deploy/yolov7-tiny.yaml: LeakyReLU convs, MP / SP pools, three-level Detect): the oracle's restatement of the
    graph against the reference's own ``Model`` (fused, eval, CPU) on the same seeded weights -- every objectness and a seeded
    sample of whole output rows, stored in tests/golden/refchecks.npz (tests/golden/make_golden_refchecks.py)."""
    from b200track import tiny
    g = np.load(REFCHECKS)
    sd = tiny.seeded_state_dict(0)
    img = torch.rand((2, 3, 192, 256), generator=torch.Generator().manual_seed(5))
    with torch.no_grad():
        got = OD.forward(tiny.tiny_layers(), sd, img, tiny.ANCHORS, tiny.STRIDES, act="leaky", name_offset=-1).double().numpy()
    assert tuple(g["tiny_shape"]) == got.shape == (2, 3 * (24 * 32 + 12 * 16 + 6 * 8), 85)
    rows = got.reshape(-1, 85)[g["tiny_row_index"]]
    assert float(np.abs(rows - g["tiny_rows"]).max()) < 2e-3 and float(np.abs(got[..., 4] - g["tiny_obj"]).max()) < 1e-5
