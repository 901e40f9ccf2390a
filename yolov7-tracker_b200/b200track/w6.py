"""YOLOv7-w6 graph (deploy form) for the H100 detector branch.

The reference builds this network from ``cfg/deploy/yolov7-w6.yaml`` through ``parse_model``
(models/yolo.py:443-520) and runs it module by module (``Model.forward_once`` :321-351).  Here the
same 119-layer DAG is generated programmatically (``w6_layers``), a planner assigns every tensor a
place in an NHWC bf16 buffer -- tensors that feed a ``Concat`` are produced straight into the concat
buffer (concat-by-address, no copy) -- and every ``Conv`` becomes one launch of the wgmma conv kernel.

Layer tuple: (index, op, from, args).  ops: 'reorg', 'conv' (cout, k, s), 'concat', 'up', 'sppcspc' (cout), 'detect'.
Weights use the reference's fused state-dict names (``model.{i}.conv.weight`` / ``.bias``,
``model.47.cv{1..7}.conv.*``, ``model.118.m.{j}.*``).
"""
import math

import torch

ANCHORS = [[19, 27, 44, 40, 38, 94], [96, 68, 86, 152, 180, 137], [140, 301, 303, 264, 238, 542], [436, 615, 739, 380, 925, 792]]
STRIDES = [8, 16, 32, 64]
NC = 80
NO = NC + 5


def w6_layers():
    L = []

    def add(op, frm, *args):
        L.append((len(L), op, frm, args))
        return len(L) - 1

    add("reorg", -1)
    add("conv", -1, 64, 3, 1)

    def elan_backbone(c_down, c_mid, c_out):
        add("conv", -1, c_down, 3, 2)
        add("conv", -1, c_mid, 1, 1)
        add("conv", -2, c_mid, 1, 1)
        for _ in range(4):
            add("conv", -1, c_mid, 3, 1)
        add("concat", [-1, -3, -5, -6])
        return add("conv", -1, c_out, 1, 1)

    p2 = elan_backbone(128, 64, 128)      # 10
    p3 = elan_backbone(256, 128, 256)     # 19
    p4 = elan_backbone(512, 256, 512)     # 28
    p5 = elan_backbone(768, 384, 768)     # 37
    elan_backbone(1024, 512, 1024)        # 46
    spp = add("sppcspc", -1, 512)         # 47

    def elan_head(c, c_half):
        add("conv", -1, c, 1, 1)
        add("conv", -2, c, 1, 1)
        for _ in range(4):
            add("conv", -1, c_half, 3, 1)
        add("concat", [-1, -2, -3, -4, -5, -6])
        return add("conv", -1, c, 1, 1)

    def up_block(c, route):
        add("conv", -1, c, 1, 1)
        add("up", -1)
        add("conv", route, c, 1, 1)
        add("concat", [-1, -2])
        return elan_head(c, c // 2)

    h5 = up_block(384, p5)                # 59
    h4 = up_block(256, p4)                # 71
    h3 = up_block(128, p3)                # 83

    def down_block(c, other):
        add("conv", -1, c, 3, 2)
        add("concat", [-1, other])
        return elan_head(c, c // 2)

    n4 = down_block(256, h4)              # 93
    n5 = down_block(384, h5)              # 103
    n6 = down_block(512, spp)             # 113
    o3 = add("conv", h3, 256, 3, 1)
    o4 = add("conv", n4, 512, 3, 1)
    o5 = add("conv", n5, 768, 3, 1)
    o6 = add("conv", n6, 1024, 3, 1)
    add("detect", [o3, o4, o5, o6])
    assert len(L) == 119 and (p2, p3, p4, p5, spp, h5, h4, h3, n4, n5, n6) == (10, 19, 28, 37, 47, 59, 71, 83, 93, 103, 113)
    return L


def _resolve(i, f):
    return f if f >= 0 else i + f


def layer_channels(layers=None, ch_in=3):
    """Output channels of every layer (the bookkeeping parse_model does, models/yolo.py:447-516)."""
    layers = layers or w6_layers()
    ch = []
    for i, op, frm, args in layers:
        if op == "reorg":
            c = ch_in * 4
        elif op == "input":
            c = ch_in
        elif op in ("mp", "sp"):
            c = ch[_resolve(i, frm)]
        elif op == "conv":
            c = args[0]
        elif op == "concat":
            c = sum(ch[_resolve(i, f)] for f in frm)
        elif op == "up":
            c = ch[_resolve(i, frm)]
        elif op == "sppcspc":
            c = args[0]
        elif op == "detect":
            c = 0
        ch.append(c)
    return ch


def stackable_pairs(layers=None):
    """[(i, i + 1)]: consecutive 1x1/s1 convs that read the SAME tensor (``from`` -1 and -2) and end up next to each other in
    the same ``Concat`` ([... | conv i+1 | conv i]) -- the two branches that open every ELAN block.  They can run as one
    convolution whose weight rows are ``cat(W[i+1], W[i])`` writing the joint slice."""
    layers = layers or w6_layers()
    ch = layer_channels(layers)
    # channel offset of every tensor inside the concat that consumes it
    where = {}
    for i, op, frm, args in layers:
        if op == "concat":
            off = 0
            for f in frm:
                j = _resolve(i, f)
                where[j] = (i, off)
                off += ch[j]
    out = []
    for (i, op, frm, args), nxt in zip(layers, layers[1:]):
        if op != "conv" or nxt[1] != "conv" or args[1:] != (1, 1) or nxt[3][1:] != (1, 1):
            continue
        if _resolve(i, frm) != _resolve(nxt[0], nxt[2]):
            continue
        a, b = where.get(i), where.get(nxt[0])
        if a and b and a[0] == b[0] and b[1] + ch[nxt[0]] == a[1]:
            out.append((i, nxt[0]))
    return out


def conv_shapes(layers=None, name_offset=0):
    """[(name, cin, cout, k, s, act)] of every fused conv, reference state-dict names (module index = layer index + name_offset)."""
    layers = layers or w6_layers()
    no_ = name_offset
    ch = layer_channels(layers)
    out = []
    for i, op, frm, args in layers:
        if op == "conv":
            out.append(("model.%d.conv" % (i + no_), ch[_resolve(i, frm)], args[0], args[1], args[2], True))
        elif op == "sppcspc":
            c1, c2 = ch[_resolve(i, frm)], args[0]
            c_ = int(2 * c2 * 0.5)
            for name, ci, co, k in (("cv1", c1, c_, 1), ("cv2", c1, c_, 1), ("cv3", c_, c_, 3), ("cv4", c_, c_, 1),
                                    ("cv5", 4 * c_, c_, 1), ("cv6", c_, c_, 3), ("cv7", 2 * c_, c2, 1)):
                out.append(("model.%d.%s.conv" % (i, name), ci, co, k, 1, True))
        elif op == "detect":
            for j, f in enumerate(frm):
                out.append(("model.%d.m.%d" % (i + no_, j), ch[f], 3 * NO, 1, 1, False))
    return out


def fold_reference_state_dict(sd, bn_eps=1e-3):
    """Any of the reference's w6 checkpoint formats -> the fused deploy-graph state dict this package runs.

    * deploy / already fused (``Model('cfg/deploy/yolov7-w6.yaml').fuse()``): ``model.{i}.conv.{weight,bias}``, head ``model.118.m.{j}``;
      returned unchanged;
    * unfused (``conv.weight`` + ``bn.*``): BatchNorm folded exactly as ``fuse_conv_and_bn`` does (utils/torch_utils.py:181-201;
      eps = 1e-3 is what ``initialize_weights`` sets, :150);
    * training graph (``cfg/training/yolov7-w6.yaml``): layers 118-121 are the auxiliary-head convs and the head is an
      ``IAuxDetect`` at index 122 (models/yolo.py:111-153).  Inference uses only ``m[j](ia[j] + x) * im[j]``, i.e. a plain 1x1
      conv with  W' = im * W,  b' = im * (b + W . ia)  (what ``IDetect.fuse`` does, :105-123 region of the upstream file): the
      implicit tensors are folded, ``m2`` and layers 118-121 are dropped, the head is renamed to ``model.118``."""
    need = {n for n, *_ in conv_shapes()}
    out = {}
    head_idx = None
    for k in sd:
        parts = k.split(".")
        if len(parts) >= 4 and parts[0] == "model" and parts[2] == "m" and parts[-1] == "weight":
            head_idx = int(parts[1])
    if head_idx is None:
        raise KeyError("no Detect head (model.<i>.m.<j>.weight) in the state dict")

    def fold_conv(prefix):
        w = sd[prefix + ".conv.weight"].float()
        if prefix + ".bn.weight" not in sd:
            return w, sd[prefix + ".conv.bias"].float()
        g, beta = sd[prefix + ".bn.weight"].float(), sd[prefix + ".bn.bias"].float()
        mu, var = sd[prefix + ".bn.running_mean"].float(), sd[prefix + ".bn.running_var"].float()
        scale = g / torch.sqrt(bn_eps + var)
        b_conv = sd[prefix + ".conv.bias"].float() if prefix + ".conv.bias" in sd else torch.zeros_like(mu)
        return w * scale.view(-1, 1, 1, 1), scale * b_conv + (beta - g * mu / torch.sqrt(var + bn_eps))

    for name in sorted(need):
        if ".m." in name:                               # Detect head j
            j = int(name.rsplit(".", 1)[1])
            src = "model.%d" % head_idx
            w, b = sd["%s.m.%d.weight" % (src, j)].float(), sd["%s.m.%d.bias" % (src, j)].float()
            ia, im = sd.get("%s.ia.%d.implicit" % (src, j)), sd.get("%s.im.%d.implicit" % (src, j))
            if ia is not None:
                b = b + (w.view(w.shape[0], -1) @ ia.float().view(-1))
            if im is not None:
                m = im.float().view(-1)
                w, b = w * m.view(-1, 1, 1, 1), b * m
        else:
            w, b = fold_conv(name[:-len(".conv")])
        out[name + ".weight"], out[name + ".bias"] = w.contiguous(), b.contiguous()
    return out


# RMS of the four Detect inputs measured once with gain = 1.68 on a seeded image (tests/golden/make_golden_detector.py);
# dividing the head weights by it gives logits of the requested spread.
HEAD_INPUT_RMS = (0.40, 0.16, 0.16, 0.125)


def seeded_state_dict(seed=0, device="cpu", gain=1.68, obj_mean=-6.5, obj_std=1.5, cls_mean=-1.0, cls_std=1.0):
    """Seeded, variance-preserving random weights in the reference's FUSED naming.

    The reference ships no detector checkpoint, and its default init makes activations vanish with
    depth (1e-13 at the neck, SURVEY 7.2 #6): NMS then sees zero candidates and every parity test is
    vacuous.  Here every conv gets N(0, gain^2 / fan_in) weights (gain ~ 1.75 keeps the post-SiLU
    second moment near 1; the network is ~60 convs deep, so the gain is tuned to 1.68) and a small bias; the Detect head is scaled so that objectness logits are
    ~ N(obj_mean, obj_std^2) -- roughly 10 % of the 102 000 anchors pass conf_thres = 0.01 and NMS hits
    its 300-detection cap.  The same dict drives the CUDA path, the torch oracle and the CPU baseline.
    """
    g = torch.Generator(device="cpu").manual_seed(seed)
    sd = {}
    for name, cin, cout, k, s, act in conv_shapes():
        fan_in = cin * k * k
        if act:
            w = torch.randn((cout, cin, k, k), generator=g) * (gain / math.sqrt(fan_in))
            b = torch.randn(cout, generator=g) * 0.1
        else:
            w = torch.randn((cout, cin, k, k), generator=g) / math.sqrt(fan_in)
            b = torch.zeros(cout)
            w /= HEAD_INPUT_RMS[int(name.rsplit(".", 1)[1])]
            wv, bv = w.view(3, NO, cin), b.view(3, NO)
            wv[:, 0:4] *= 1.0
            wv[:, 4] *= obj_std
            wv[:, 5:] *= cls_std
            bv[:, 4] = obj_mean
            bv[:, 5:] = cls_mean
        sd[name + ".weight"] = w.to(device)
        sd[name + ".bias"] = b.to(device)
    return sd


def calibrated_state_dict(seed=0, img_size=1280, device="cuda", obj_mean=-6.5, obj_std=1.5, cls_mean=-1.0, cls_std=1.0, img=None, act_std=1.0):
    """``seeded_state_dict`` followed by a layer-sequential, data-dependent rescale (LSUV style): every conv's
    weights are divided by the measured std of its pre-activation on a seeded image of the requested size, and the
    Detect rows are scaled to the requested logit spreads.  A fixed gain cannot do this: the net is ~60 convs deep and
    the critical gain depends on the resolution (zero-padded borders), so at 1280 x 1280 the plain seeded weights blow
    up (80 % of the anchors pass conf_thres) while at 256 x 256 they are fine.  Init-time plumbing in plain torch
    (fp32); returns the fused-name state dict that the CUDA path, the oracle and the CPU baseline all load.
    ``act_std``: pre-activation standard deviation every conv is scaled to.  1.0 (default, the bench weights) puts SiLU in its
    non-linear range: a random 60-layer net then amplifies a 1e-4 perturbation ~30x by the head (chaotic regime).  0.5 keeps SiLU close to linear -- perturbations are not amplified -- and is what the
    tight detector-parity test uses to tell kernel errors from the network's own sensitivity."""
    import torch.nn.functional as F
    sd = {k: v.to(device) for k, v in seeded_state_dict(seed).items()}
    if img is None:
        g = torch.Generator(device="cpu").manual_seed(seed + 1000)
        img = torch.rand((1, 3, img_size, img_size), generator=g)
    x0 = img.to(device).float()
    layers = w6_layers()
    y = []

    def conv(name, x, k, s, act=True):
        w, b = sd[name + ".weight"], sd[name + ".bias"]
        z = F.conv2d(x, w, None, stride=s, padding=k // 2)
        if act:
            w /= z.std().clamp_min(1e-6) / act_std
            z = F.conv2d(x, w, b, stride=s, padding=k // 2)
            return z * torch.sigmoid(z)
        # Detect rows: box / objectness / class groups get their own spread
        cout = w.shape[0]
        zz = z.view(z.shape[0], 3, NO, -1)
        wv, bv = w.view(3, NO, -1), b.view(3, NO)
        for sl, std, mean in ((slice(0, 4), 1.0, 0.0), (slice(4, 5), obj_std, obj_mean), (slice(5, NO), cls_std, cls_mean)):
            wv[:, sl] *= std / zz[:, :, sl].std().clamp_min(1e-6)
            bv[:, sl] = mean
        return None

    with torch.no_grad():
        for i, op, frm, args in layers:
            if op == "reorg":
                out = torch.cat([x0[..., ::2, ::2], x0[..., 1::2, ::2], x0[..., ::2, 1::2], x0[..., 1::2, 1::2]], 1)
            elif op == "conv":
                out = conv("model.%d.conv" % i, y[_resolve(i, frm)], args[1], args[2])
            elif op == "concat":
                out = torch.cat([y[_resolve(i, f)] for f in frm], 1)
            elif op == "up":
                out = F.interpolate(y[_resolve(i, frm)], scale_factor=2, mode="nearest")
            elif op == "sppcspc":
                xin = y[_resolve(i, frm)]
                p = "model.%d." % i
                x1 = conv(p + "cv4.conv", conv(p + "cv3.conv", conv(p + "cv1.conv", xin, 1, 1), 3, 1), 1, 1)
                pools = [F.max_pool2d(x1, k, 1, k // 2) for k in (5, 9, 13)]
                y1 = conv(p + "cv6.conv", conv(p + "cv5.conv", torch.cat([x1] + pools, 1), 1, 1), 3, 1)
                y2 = conv(p + "cv2.conv", xin, 1, 1)
                out = conv(p + "cv7.conv", torch.cat((y1, y2), 1), 1, 1)
            elif op == "detect":
                for lvl, f in enumerate(frm):
                    conv("model.%d.m.%d" % (i, lvl), y[f], 1, 1, act=False)
                break
            y.append(out)
            # free tensors nobody needs any more (1280^2 activations are large in fp32)
    return sd
