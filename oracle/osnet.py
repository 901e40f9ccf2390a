"""TEST INFRASTRUCTURE ONLY -- CPU restatement of StrongSORT's appearance network (tracker/strongsort.py:26-29, :47-89;
tracker/reid_models/OSNet.py ``osnet_x0_25``).

``preprocess`` restates ``StrongSORT.reid_preprocess`` :47-64 in NumPy: crop.astype(float32) / 255 -> cv2.resize(dsize=(256, 128)) ->
ToTensor -> Normalize.  cv2's dsize is (width, height), so the network sees 128 rows x 256 columns; ``size`` is (rows, columns).
``forward`` restates ``OSNet.forward`` in eval mode (the extractor is ``.eval()``-ed, strongsort.py:28) with torch.nn.functional on a
state dict: BatchNorm with the running statistics, unfolded.  tests/test_oracle_osnet.py pins both against the UNMODIFIED reference
(tests/golden/osnet.npz, made by tests/golden/make_golden_osnet.py).
"""
import functools

import numpy as np
import torch
import torch.nn.functional as F

from .reid import MEAN, STD, _taps, seeded_crops

CHANNELS = (16, 64, 96, 128)
FEATURE_DIM = 512
# stage -> (input channels, output channels, has a transition (Conv1x1 + AvgPool 2 x 2))
STAGES = (("conv2", 16, 64, True), ("conv3", 64, 96, True), ("conv4", 96, 128, False))
STREAMS = (("conv2a", 1), ("conv2b", 2), ("conv2c", 3), ("conv2d", 4))
EPS = 1e-5


def preprocess(crops, size=(128, 256)):
    """list of (h, w, 3) uint8 BGR -> (n, 3, size[0], size[1]) float32 tensor."""
    oh, ow = size
    out = []
    for im in crops:
        a = im.astype(np.float32) / np.float32(255.0)
        h, w = a.shape[:2]
        x0, x1, fx = _taps(ow, w)
        y0, y1, fy = _taps(oh, h)
        fx = fx[None, :, None]; fy = fy[:, None, None]
        rows = a[:, x0] * (np.float32(1) - fx) + a[:, x1] * fx
        r = rows[y0] * (np.float32(1) - fy) + rows[y1] * fy
        r = (r - MEAN) / STD                                       # Normalize on the channels as they come (B, G, R)
        out.append(torch.from_numpy(np.ascontiguousarray(r.transpose(2, 0, 1))))
    return torch.stack(out).float()


def block_names():
    """(prefix, cin, cout) of the six OSBlocks in order."""
    out = []
    for stage, cin, cout, _ in STAGES:
        out += [("%s.0" % stage, cin, cout), ("%s.1" % stage, cout, cout)]
    return out


def state_dict_shapes(num_classes=1):
    """The keys and shapes of osnet_x0_25(num_classes)'s state dict, in the module's registration order."""
    shapes = []

    def bn(p, c):
        shapes.extend([(p + ".weight", (c,)), (p + ".bias", (c,)), (p + ".running_mean", (c,)), (p + ".running_var", (c,)),
                       (p + ".num_batches_tracked", ())])

    def conv_bn(p, cout, cin, k=1):
        shapes.append((p + ".conv.weight", (cout, cin, k, k)))
        bn(p + ".bn", cout)

    def light(p, c):
        shapes.extend([(p + ".conv1.weight", (c, c, 1, 1)), (p + ".conv2.weight", (c, 1, 3, 3))])
        bn(p + ".bn", c)

    conv_bn("conv1", 16, 3, 7)
    for stage, cin, cout, trans in STAGES:
        for blk in range(2):
            p, ci = "%s.%d" % (stage, blk), (cin if blk == 0 else cout)
            mid = cout // 4
            conv_bn(p + ".conv1", mid, ci)
            light(p + ".conv2a", mid)
            for name, k in STREAMS[1:]:
                for i in range(k):
                    light("%s.%s.%d" % (p, name, i), mid)
            hid = mid // 16
            shapes.extend([(p + ".gate.fc1.weight", (hid, mid, 1, 1)), (p + ".gate.fc1.bias", (hid,)),
                           (p + ".gate.fc2.weight", (mid, hid, 1, 1)), (p + ".gate.fc2.bias", (mid,))])
            conv_bn(p + ".conv3", cout, mid)
            if ci != cout:
                conv_bn(p + ".downsample", cout, ci)
        if trans:
            conv_bn("%s.2.0" % stage, cout, cout)
    conv_bn("conv5", 128, 128)
    shapes.extend([("fc.0.weight", (FEATURE_DIM, 128)), ("fc.0.bias", (FEATURE_DIM,))])
    bn("fc.1", FEATURE_DIM)
    shapes.extend([("classifier.weight", (num_classes, FEATURE_DIM)), ("classifier.bias", (num_classes,))])
    return shapes


class _BN:
    """BatchNorm with the running statistics; calibrate=True first sets them to the statistics of the input it sees (float64)."""
    calibrate = False


def _bn(x, sd, p):
    if _BN.calibrate:
        dims = [d for d in range(x.dim()) if d != 1]
        sd[p + ".running_mean"] = x.mean(dims).to(sd[p + ".running_mean"].dtype)
        # a floor at the layer's mean variance: a nearly dead channel must not get a huge folded scale (the real checkpoint has none)
        v = x.var(dims, unbiased=False)
        sd[p + ".running_var"] = (v.mean() + 0.3 * v).to(sd[p + ".running_var"].dtype)
    return F.batch_norm(x, sd[p + ".running_mean"], sd[p + ".running_var"], sd[p + ".weight"], sd[p + ".bias"], False, 0.0, EPS)


def _conv_bn(x, sd, p, relu=True, stride=1, padding=0):
    y = _bn(F.conv2d(x, sd[p + ".conv.weight"], None, stride, padding), sd, p + ".bn")
    return F.relu(y) if relu else y


def _light(x, sd, p):
    y = F.conv2d(x, sd[p + ".conv1.weight"])
    y = F.conv2d(y, sd[p + ".conv2.weight"], None, 1, 1, 1, y.shape[1])
    return F.relu(_bn(y, sd, p + ".bn"))


def gate_values(x, sd, p):
    """ChannelGate's sigmoid outputs (n, c) for one stream x."""
    g = x.mean((2, 3), keepdim=True)
    g = F.relu(F.conv2d(g, sd[p + ".fc1.weight"], sd[p + ".fc1.bias"]))
    return torch.sigmoid(F.conv2d(g, sd[p + ".fc2.weight"], sd[p + ".fc2.bias"])).flatten(1)


def streams(x1, sd, p):
    """The four LightConv3x3 streams of OSBlock p on x1."""
    out = []
    for name, k in STREAMS:
        y = x1
        for i in range(k):
            y = _light(y, sd, ("%s.%s" % (p, name)) if k == 1 else ("%s.%s.%d" % (p, name, i)))
        out.append(y)
    return out


def block(x, sd, p, trace=None):
    x1 = _conv_bn(x, sd, p + ".conv1")
    ss = streams(x1, sd, p)
    gates = [gate_values(s, sd, p + ".gate") for s in ss]
    x2 = ss[0] * gates[0][:, :, None, None]
    for s, g in zip(ss[1:], gates[1:]):
        x2 = x2 + s * g[:, :, None, None]
    if trace is not None:
        trace.append((p, gates))
    x3 = _conv_bn(x2, sd, p + ".conv3", relu=False)
    idn = _conv_bn(x, sd, p + ".downsample", relu=False) if (p + ".downsample.conv.weight") in sd else x
    return F.relu(x3 + idn)


def forward(sd, x, trace=None):
    """OSNet.forward in eval mode: (n, 3, H, W) -> (n, 512) (after fc's ReLU, not normalised).  trace: a list that receives
    (block prefix, [gate values of the four streams]) per OSBlock."""
    x = _conv_bn(x, sd, "conv1", stride=2, padding=3)
    x = F.max_pool2d(x, 3, 2, 1)
    for stage, _, _, trans in STAGES:
        for blk in range(2):
            x = block(x, sd, "%s.%d" % (stage, blk), trace)
        if trans:
            x = F.avg_pool2d(_conv_bn(x, sd, "%s.2.0" % stage), 2, 2)
    x = _conv_bn(x, sd, "conv5")
    v = x.mean((2, 3))
    v = F.linear(v, sd["fc.0.weight"], sd["fc.0.bias"])
    return F.relu(_bn(v, sd, "fc.1"))


@functools.lru_cache(maxsize=8)
def _seeded(seed, num_classes):
    g = torch.Generator().manual_seed(seed)
    sd = {}
    for k, shape in state_dict_shapes(num_classes):
        if k.endswith("num_batches_tracked"):
            sd[k] = torch.zeros((), dtype=torch.int64)
        elif k.endswith(".running_mean"):
            sd[k] = torch.zeros(shape, dtype=torch.float64)
        elif k.endswith(".running_var"):
            sd[k] = torch.ones(shape, dtype=torch.float64)
        elif k.endswith("bn.weight") or k == "fc.1.weight":
            sd[k] = 0.4 + 0.6 * torch.rand(shape, generator=g, dtype=torch.float64)
        elif k.endswith("bn.bias"):
            sd[k] = 0.2 * torch.randn(shape, generator=g, dtype=torch.float64)
        elif k == "fc.1.bias":
            sd[k] = 0.3 + 0.5 * torch.randn(shape, generator=g, dtype=torch.float64)
        elif k.endswith(".bias"):                               # gate fc biases, fc.0, classifier
            sd[k] = 0.1 * torch.randn(shape, generator=g, dtype=torch.float64)
        else:                                                   # conv / linear weights: variance 1 / fan_in (the gates' wider,
            fan_in = int(np.prod(shape[1:]))                    # so that their sigmoids differ from stream to stream)
            sd[k] = torch.randn(shape, generator=g, dtype=torch.float64) * ((3.0 if ".gate." in k else 1.0) / fan_in ** 0.5)
    # running statistics: those of seeded crops at the reference's 128 x 256, layer by layer (float64), so that every BatchNorm
    # normalises for real and the activations stay O(1) through the 16 blocks
    x = preprocess(seeded_crops(seed + 1000, 8)).double()
    _BN.calibrate = True
    try:
        with torch.no_grad():
            forward(sd, x)
    finally:
        _BN.calibrate = False
    return {k: (v.float() if v.is_floating_point() else v) for k, v in sd.items()}


def seeded_state_dict(seed=0, num_classes=1):
    """A float32 state dict with the keys and shapes of osnet_x0_25(num_classes): weights of variance 1 / fan_in, BatchNorm affine
    parameters away from the identity and running statistics calibrated on seeded crops."""
    return {k: v.clone() for k, v in _seeded(int(seed), int(num_classes)).items()}
