"""not-gpu: the launch plan DetectorW6 builds (every conv descriptor, the op order, the head levels), recorded on CPU by
tests/plan_dryrun.py, against (a) the committed plan of the build that passed the round-1 GPU parity tests
(tests/golden/w6_plan.json) and (b) for non-square inputs, the tensor shapes of the torch oracle."""
import json
import os
import sys

import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from plan_dryrun import dry_run_plan  # noqa: E402

GOLDEN = os.path.join(os.path.dirname(__file__), "golden", "w6_plan.json")


def _norm(conv):
    return {k: (list(v) if isinstance(v, (list, tuple)) else v) for k, v in conv.items()}


@pytest.mark.parametrize("idx", [0, 1])
def test_square_plan_equals_gpu_verified_golden(idx):
    g = json.load(open(GOLDEN))[idx]
    det, plan = dry_run_plan(g["batch"], g["size"])
    assert det.n_total == g["n_total"] and [n for _, _, n in det.ops] == g["ops"]
    assert len(plan) == len(g["convs"]) == 96
    for k, (a, b) in enumerate(zip(plan, g["convs"])):
        assert _norm(a) == b, "conv %d (%s) differs from the verified plan" % (k, g["ops"][k])
    assert det.launch_log == g["launches"]                              # scalar arguments of every glue / decode / NMS call
    for lv, ref in zip(det.head_levels, g["levels"]):
        assert (lv.h, lv.w, lv.stride, lv.level_off, lv.raw_pitch, list(lv.anchors)) == (ref["h"], ref["w"], ref["stride"], ref["level_off"],
                                                                                          ref["raw_pitch"], ref["anchors"])


def test_non_square_plan_matches_oracle_shapes():
    """(H, W) = (256, 384): every tensor the planner lays out has the size the torch oracle produces, the prediction rows are
    numbered level by level as Detect.forward concatenates them, and NMS clips to (W, H)."""
    from b200track.w6 import ANCHORS, STRIDES, seeded_state_dict, w6_layers
    from oracle import detector as OD
    H, W = 256, 384
    det, plan = dry_run_plan(1, (H, W))
    with torch.no_grad():
        pred, raw = OD.forward(w6_layers(), seeded_state_dict(0), torch.zeros((1, 3, H, W)), ANCHORS, STRIDES, return_raw=True)
    assert det.n_total == pred.shape[1] and tuple(det.pred.shape) == tuple(pred.shape)
    off = 0
    for lv, r in zip(det.head_levels, raw):                          # raw: (B, 3, h, w, 85)
        assert (lv.h, lv.w) == (r.shape[2], r.shape[3]) and lv.level_off == off
        off += 3 * lv.h * lv.w
    assert tuple(det.img.shape) == (1, 3, H, W) and det.S is None
    # stem reads the padded ReOrg buffer; every conv's output buffer is (1, ho, wo, pitch) with ho / wo = input / stride
    assert plan[0]["x_shape"] == [1, H // 2, W // 2 + 8, 16] and plan[0]["in_row_pixels"] == W // 2 + 8
    for c in plan:
        assert c["y_shape"][1] == c["h"] // c["stride"] and c["y_shape"][2] == c["w"] // c["stride"]
        assert c["h"] * 3 == c["w"] * 2                              # the 2:3 aspect ratio survives every stride
    calls = {l[0]: l for l in det.launch_log}
    assert calls["b2t_image_reorg_padded"][3:8] == [1, H, W, W // 2 + 8, 1]
    nms = calls["b2t_detect_nms"]
    assert nms[-7:-5] == [float(W), float(H)]                         # img_w, img_h of scale_coords / clip_coords
    up = [l for l in det.launch_log if l[0] == "b2t_upsample2x"]
    assert all(l[8] * 3 == l[9] * 2 for l in up)                      # (B, H, W) of every upsample keeps the ratio


def test_plan_960x1280_stride_64_rectangle():
    """A 4:3 source letterboxed with stride 64 (tracker_dataloader.py:100-126) is 960 x 1280: not a multiple of 128, planned all the
    same (P6 map 15 x 20); shapes follow the oracle's."""
    from b200track.w6 import ANCHORS, STRIDES, seeded_state_dict, w6_layers
    from oracle import detector as OD
    H, W = 960, 1280
    det, plan = dry_run_plan(1, (H, W))
    assert [(lv.h, lv.w) for lv in det.head_levels] == [(120, 160), (60, 80), (30, 40), (15, 20)]
    assert det.n_total == 3 * (120 * 160 + 60 * 80 + 30 * 40 + 15 * 20)
    for c in plan:
        assert c["y_shape"][1] == (c["h"] + c["stride"] - 1) // c["stride"] and c["y_shape"][2] == (c["w"] + c["stride"] - 1) // c["stride"]


def test_tiny_plan_structure_on_cpu():
    """The YOLOv7-tiny planner (b200track/tiny.py) dry-run on CPU tensors: 58 convs in 50 launches (8 stacked ELAN pairs), LeakyReLU
    on all but the three Detect convs, three MP launches, one launch for the three SP pools, the SPP concat stored as [x | m5 | m9 | m13]
    with the consuming conv's input channels permuted from the reference's [m13 | m9 | m5 | x], output maps of the oracle's shapes."""
    import ctypes as C  # noqa: F401
    from collections import Counter
    from unittest import mock

    import torch
    from plan_dryrun import RecorderLib
    from b200track import _lib as L
    from b200track import tiny
    from oracle import detector as OD
    rec = RecorderLib()
    with mock.patch.object(L, "load", lambda: rec), mock.patch.object(torch.cuda, "is_available", lambda: True):
        det = tiny.DetectorTiny(tiny.seeded_state_dict(0), batch=2, img_size=(192, 256), device="cpu", use_graph=False, autotune=False)
    rec.launches = []

    class _S:
        cuda_stream = 0
    with mock.patch.object(torch.cuda, "current_stream", lambda *a, **k: _S()):
        det._forward_launches(); det.decode(); det._nms_launch(True)
    names = Counter(l[0] for l in rec.launches)
    assert names["b2t_conv_run"] == 50 and names["b2t_maxpool2x2s2"] == 3 and names["b2t_spp_pool"] == 1 and names["b2t_upsample2x"] == 2
    assert names["b2t_image_nhwc16"] == 1 and names["b2t_detect_decode"] == 3 and names["b2t_detect_nms"] == 1
    assert Counter(d["act"] for d in rec.descs) == {3: 47, 0: 3}
    assert rec.descs[0]["cin"] == 16 and rec.descs[0]["stride"] == 2 and rec.descs[0]["cout"] == 32          # the image conv: 3 -> 16 padded channels
    (ci, perm), = det.in_perm.items()
    assert perm.tolist() == list(range(768, 1024)) + list(range(512, 768)) + list(range(256, 512)) + list(range(0, 256))
    with torch.no_grad():
        pred = OD.forward(tiny.tiny_layers(), tiny.seeded_state_dict(0), torch.zeros((2, 3, 192, 256)), tiny.ANCHORS, tiny.STRIDES, act="leaky", name_offset=-1)
    assert det.n_total == pred.shape[1] == 3 * (24 * 32 + 12 * 16 + 6 * 8)
    assert [tuple(r.shape) for r in det.raw] == [(2, 24, 32, 256), (2, 12, 16, 256), (2, 6, 8, 256)]
