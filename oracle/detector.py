"""Oracle: YOLOv7 forward / decode / NMS restated in plain PyTorch fp32.

TEST INFRASTRUCTURE (see oracle/__init__.py).  Executes a layer list of the form produced by the
product's graph builder -- (index, op, from, args) with ops reorg / conv / concat / up / sppcspc /
detect -- with ``torch.nn.functional`` on NCHW fp32 tensors, following
  Model.forward_once      models/yolo.py:321-351      ReOrg / Concat / SPPCSPC   models/common.py:48-62, 262-280
  Conv.fuseforward        models/common.py:110-111    Detect.forward             models/yolo.py:39-57
  non_max_suppression     utils/general.py:607-695 (best-class path) with torchvision.ops.nms
Pinned against the reference's own ``Model('cfg/deploy/yolov7-w6.yaml')`` loaded with the same seeded
weights in the build container (tests/golden/detector_w6.npz, tests/golden/make_golden_detector.py).
``emulate_bf16`` (True = bfloat16, or torch.float16 / torch.bfloat16) rounds weights and every conv output to the
16-bit type the tensor-core path stores them in (16-bit operands, fp32 accumulation) -- to separate kernel bugs from
precision effects.
"""
import torch
import torch.nn.functional as F


def _r(i, f):
    return f if f >= 0 else i + f


def _bf(t, on):
    """on: False / None = exact fp32, True = bfloat16, or a torch dtype (torch.float16 / torch.bfloat16): round to the 16-bit
    type the tensor-core path stores activations and weights in."""
    if not on:
        return t
    return t.to(torch.bfloat16 if on is True else on).float()


def forward(layers, sd, img, anchors, strides, nc=80, emulate_bf16=False, return_raw=False, act="silu", name_offset=0, return_layers=False):
    """img (B,3,H,W) float32 in [0,1] -> pred (B, N, 5+nc) as ``model(img)[0]`` of the fused reference model.
    act: "silu" (w6, models/common.py:105) or "leaky" (YOLOv7-tiny: nn.LeakyReLU(0.1), cfg/deploy/yolov7-tiny.yaml:15);
    name_offset: layer index -> the reference's module index (the tiny layer list carries an explicit input op in front: -1).
    return_layers: return dict(pred, layers = every layer's output by index (None for Detect), spp = {layer index: the SPPCSPC
    temporaries t1 (cv1), t2 (cv3), x1 (cv4), m5 / m9 / m13 (pools of x1), t5 (cv5), y1 (cv6), y2 (cv2)}, raw = the Detect
    convs' (B, 3 * no, h, w) outputs per level) -- a chain of stored layer outputs to check a per-layer harness against."""
    no = nc + 5
    no_ = name_offset
    dev = img.device
    y = []
    spp = {}

    def conv(name, x, k, s, act=True):
        w = _bf(sd[name + ".weight"].to(dev).float(), emulate_bf16)
        b = sd[name + ".bias"].to(dev).float()
        o = F.conv2d(x, w, b, stride=s, padding=k // 2)
        if act:
            o = o * torch.sigmoid(o) if globals_act[0] == "silu" else F.leaky_relu(o, 0.1)
            o = _bf(o, emulate_bf16)
        return o

    globals_act = [act]
    x = _bf(img.float(), emulate_bf16)
    for i, op, frm, args in layers:
        if op == "input":
            out = x
        elif op == "mp":                                          # MP: nn.MaxPool2d(2, 2), models/common.py:30-35
            out = F.max_pool2d(y[_r(i, frm)], 2, 2)
        elif op == "sp":                                          # SP: nn.MaxPool2d(k, 1, k // 2), models/common.py:38-45
            out = F.max_pool2d(y[_r(i, frm)], args[0], 1, args[0] // 2)
        elif op == "reorg":
            src = x
            out = torch.cat([src[..., ::2, ::2], src[..., 1::2, ::2], src[..., ::2, 1::2], src[..., 1::2, 1::2]], 1)
        elif op == "conv":
            out = conv("model.%d.conv" % (i + no_), y[_r(i, frm)], args[1], args[2])
        elif op == "concat":
            out = torch.cat([y[_r(i, f)] for f in frm], 1)
        elif op == "up":
            out = F.interpolate(y[_r(i, frm)], scale_factor=2, mode="nearest")
        elif op == "sppcspc":
            xin = y[_r(i, frm)]
            p = "model.%d." % (i + no_)
            t1 = conv(p + "cv1.conv", xin, 1, 1)
            t2 = conv(p + "cv3.conv", t1, 3, 1)
            x1 = conv(p + "cv4.conv", t2, 1, 1)
            pools = [F.max_pool2d(x1, k, 1, k // 2) for k in (5, 9, 13)]
            t5 = conv(p + "cv5.conv", torch.cat([x1] + pools, 1), 1, 1)
            y1 = conv(p + "cv6.conv", t5, 3, 1)
            y2 = conv(p + "cv2.conv", xin, 1, 1)
            out = conv(p + "cv7.conv", torch.cat((y1, y2), 1), 1, 1)
            spp[i] = dict(t1=t1, t2=t2, x1=x1, m5=pools[0], m9=pools[1], m13=pools[2], t5=t5, y1=y1, y2=y2)
        elif op == "detect":
            z, raws, maps = [], [], []
            for lvl, f in enumerate(frm):
                r = conv("model.%d.m.%d" % (i + no_, lvl), y[f], 1, 1, act=False)
                maps.append(r)
                bs, _, ny, nx = r.shape
                r = r.view(bs, 3, no, ny, nx).permute(0, 1, 3, 4, 2).contiguous()
                raws.append(r)
                yv, xv = torch.meshgrid([torch.arange(ny, device=dev), torch.arange(nx, device=dev)], indexing="ij")
                grid = torch.stack((xv, yv), 2).view(1, 1, ny, nx, 2).float()
                a = torch.tensor(anchors[lvl], device=dev).float().view(1, 3, 1, 1, 2)
                s = r.sigmoid()
                s[..., 0:2] = (s[..., 0:2] * 2. - 0.5 + grid) * strides[lvl]
                s[..., 2:4] = (s[..., 2:4] * 2) ** 2 * a
                z.append(s.view(bs, -1, no))
            pred = torch.cat(z, 1)
            if return_layers:
                return dict(pred=pred, layers=y + [None], spp=spp, raw=maps)
            return (pred, raws) if return_raw else pred
        y.append(out)
    raise RuntimeError("layer list has no detect layer")


def seeded_training_state_dict(keys, shapes, seed):
    """A seeded state dict for a reference graph given its key names and shapes (no reference code needed): conv weights and
    biases uniform in +-1/sqrt(fan_in) (torch's default init), BatchNorm statistics / affine randomised, ImplicitA ~ N(0, 0.02),
    ImplicitM ~ N(1, 0.02), num_batches_tracked 0.  Keys are filled in the given order from ONE generator."""
    g = torch.Generator().manual_seed(int(seed))
    shapes = {k: tuple(int(v) for v in s) for k, s in zip(keys, shapes)}
    sd = {}
    for k in keys:
        shp = shapes[k]
        if k.endswith("num_batches_tracked"):
            sd[k] = torch.zeros(shp, dtype=torch.int64)
        elif k.endswith("running_mean"):
            sd[k] = torch.randn(shp, generator=g) * 0.1
        elif k.endswith("running_var"):
            sd[k] = torch.rand(shp, generator=g) * 0.5 + 0.75
        elif ".bn." in k and k.endswith(".weight"):
            sd[k] = torch.rand(shp, generator=g) * 0.5 + 1.2
        elif ".bn." in k and k.endswith(".bias"):
            sd[k] = torch.randn(shp, generator=g) * 0.1
        elif ".ia." in k:
            sd[k] = torch.randn(shp, generator=g) * 0.02
        elif ".im." in k:
            sd[k] = 1.0 + torch.randn(shp, generator=g) * 0.02
        else:
            w = shapes.get(k[:-len(".bias")] + ".weight") if k.endswith(".bias") else shp
            fan_in = int(torch.tensor(w[1:]).prod()) if w is not None and len(w) > 1 else 1
            sd[k] = (torch.rand(shp, generator=g) * 2 - 1) / fan_in ** 0.5
    return sd


def non_max_suppression(prediction, conf_thres=0.25, iou_thres=0.45, max_det=300, max_nms=30000, max_wh=4096):
    """utils/general.py:607-695, best-class branch (multi_label False, classes None, agnostic False)."""
    import torchvision
    out = [torch.zeros((0, 6), device=prediction.device)] * prediction.shape[0]
    xc = prediction[..., 4] > conf_thres
    for xi, x in enumerate(prediction):
        x = x[xc[xi]].clone()
        if not x.shape[0]:
            continue
        x[:, 5:] *= x[:, 4:5]
        box = x[:, :4].clone()
        box[:, 0] = x[:, 0] - x[:, 2] / 2
        box[:, 1] = x[:, 1] - x[:, 3] / 2
        box[:, 2] = x[:, 0] + x[:, 2] / 2
        box[:, 3] = x[:, 1] + x[:, 3] / 2
        conf, j = x[:, 5:].max(1, keepdim=True)
        x = torch.cat((box, conf, j.float()), 1)[conf.view(-1) > conf_thres]
        n = x.shape[0]
        if not n:
            continue
        if n > max_nms:
            x = x[x[:, 4].argsort(descending=True)[:max_nms]]
        c = x[:, 5:6] * max_wh
        keep = torchvision.ops.nms(x[:, :4] + c, x[:, 4], iou_thres)
        out[xi] = x[keep[:max_det]]
    return out


def post_process(det, img_hw):
    """tracker/track.py:239-240 for same-size images: scale_coords (gain 1, pad 0) + clip + round."""
    d = det.clone()
    d[:, [0, 2]] = d[:, [0, 2]].clamp(0, img_hw[1])
    d[:, [1, 3]] = d[:, [1, 3]].clamp(0, img_hw[0])
    d[:, :4] = d[:, :4].round()
    return d
