"""YOLOv7-tiny (deploy form) on the H100 detector branch -- BASELINE.json configs[0] names it.

The reference builds it from ``cfg/deploy/yolov7-tiny.yaml`` (77 modules + Detect): ``Conv`` with ``nn.LeakyReLU(0.1)`` (:15),
``MP`` = 2 x 2 max-pool (models/common.py:30-35), ``SP`` = stride-1 max-pools 5 / 9 / 13 (:38-45), ``Concat``, ``nn.Upsample``, and a
three-level ``Detect`` (strides 8 / 16 / 32).  Same planner and kernels as the w6 graph (``DetectorW6``): every conv one launch of the
wgmma conv kernel (LeakyReLU in the epilogue: act = 3), concat by address, the three SP pools one launch, MP one element-wise kernel.
Layer tuples as in ``w6.py``; index 0 is an explicit ``input`` op (float image -> NHWC 16-bit), so layer i is the reference's module i - 1.
"""
from .detector import DetectorW6

ANCHORS = [[10, 13, 16, 30, 33, 23], [30, 61, 62, 45, 59, 119], [116, 90, 156, 198, 373, 326]]
STRIDES = [8, 16, 32]
ACT_LEAKY = 3


def tiny_layers():
    """cfg/deploy/yolov7-tiny.yaml:13-111, one tuple per module (+ the input op in front): absolute ``from`` indices are shifted by one."""
    L = []

    def add(op, frm, *args):
        L.append((len(L), op, frm, args))
        return len(L) - 1

    R = lambda ref: ref + 1                                    # noqa: E731  reference module index -> index in this list

    add("input", -1)
    add("conv", -1, 32, 3, 2)                                  # 0-P1/2
    add("conv", -1, 64, 3, 2)                                  # 1-P2/4

    def elan(c, c_out):
        add("conv", -1, c, 1, 1)
        add("conv", -2, c, 1, 1)
        add("conv", -1, c, 3, 1)
        add("conv", -1, c, 3, 1)
        add("concat", [-1, -2, -3, -4])
        return add("conv", -1, c_out, 1, 1)

    elan(32, 64)                                               # 7
    add("mp", -1)                                              # 8-P3/8
    p3 = elan(64, 128)                                         # 14
    add("mp", -1)                                              # 15-P4/16
    p4 = elan(128, 256)                                        # 21
    add("mp", -1)                                              # 22-P5/32
    elan(256, 512)                                             # 28
    # head: SPP
    add("conv", -1, 256, 1, 1)                                 # 29
    add("conv", -2, 256, 1, 1)                                 # 30
    add("sp", -1, 5)
    add("sp", -2, 9)
    add("sp", -3, 13)
    add("concat", [-1, -2, -3, -4])                            # 34
    add("conv", -1, 256, 1, 1)
    add("concat", [-1, -7])
    n5 = add("conv", -1, 256, 1, 1)                            # 37
    add("conv", -1, 128, 1, 1)
    add("up", -1)
    add("conv", p4, 128, 1, 1)                                 # route backbone P4
    add("concat", [-1, -2])
    n4 = elan(64, 128)                                         # 47
    add("conv", -1, 64, 1, 1)
    add("up", -1)
    add("conv", p3, 64, 1, 1)                                  # route backbone P3
    add("concat", [-1, -2])
    n3 = elan(32, 64)                                          # 57
    add("conv", -1, 128, 3, 2)
    add("concat", [-1, n4])
    m4 = elan(64, 128)                                         # 65
    add("conv", -1, 256, 3, 2)
    add("concat", [-1, n5])
    m5 = elan(128, 256)                                        # 73
    o3 = add("conv", n3, 128, 3, 1)
    o4 = add("conv", m4, 256, 3, 1)
    o5 = add("conv", m5, 512, 3, 1)
    add("detect", [o3, o4, o5])
    assert len(L) == 79 and (p3, p4, n5, n4, n3, m4, m5) == (R(14), R(21), R(37), R(47), R(57), R(65), R(73))
    return L


def DetectorTiny(state_dict, **kw):
    """``DetectorW6`` planned for the YOLOv7-tiny graph.  state_dict: the reference's fused names (``model.{i}.conv.weight/bias``,
    ``model.77.m.{j}.*``).  The float-tensor entry points (``forward`` / ``detect`` / ``decode``); image sides multiples of 32."""
    kw.setdefault("fuse_pairs", True)
    return DetectorW6(state_dict, layers=tiny_layers(), anchors=ANCHORS, strides=STRIDES, act=ACT_LEAKY, total_stride=32, name_offset=-1, **kw)


def seeded_state_dict(seed=0, gain=1.4, obj_mean=-5.0, obj_std=1.5, cls_mean=-1.0, cls_std=1.0):
    """Seeded weights in the reference's fused naming for the tiny graph: N(0, gain^2 / fan_in) convs (gain ~ sqrt(2 / 1.01) keeps the
    post-LeakyReLU second moment), a Detect head whose objectness logits spread around obj_mean.  The reference ships no tiny checkpoint."""
    import math

    import torch
    from .w6 import NO, conv_shapes
    g = torch.Generator(device="cpu").manual_seed(seed)
    sd = {}
    for name, cin, cout, k, s, act in conv_shapes(tiny_layers(), name_offset=-1):
        fan_in = cin * k * k
        if act:
            sd[name + ".weight"] = torch.randn((cout, cin, k, k), generator=g) * (gain / math.sqrt(fan_in))
            sd[name + ".bias"] = torch.randn(cout, generator=g) * 0.1
        else:
            w = torch.randn((cout, cin, k, k), generator=g) / math.sqrt(fan_in)
            b = torch.zeros(cout)
            for a in range(3):
                w[a * NO + 4] *= obj_std; b[a * NO + 4] = obj_mean
                w[a * NO + 5:(a + 1) * NO] *= cls_std; b[a * NO + 5:(a + 1) * NO] = cls_mean
                w[a * NO:a * NO + 4] *= 0.5
            sd[name + ".weight"], sd[name + ".bias"] = w, b
    return sd
