"""-m gpu: StrongSORT's OSNet x0.25 on the kernels of csrc/b2t_osnet.cu.  Each kernel through the C ABI against its float64 reference
(tests/osnet_kernel_ref.py) at every stage geometry of 128 x 256 and 256 x 128 inputs, both 16-bit types, NaN-filled outputs fenced by
sentinels.  Then the extractor (b200track/osnet.py) against the fp32 oracle (oracle/osnet.py) per crop -- cosine >= 0.9999 and relative
L2 <= 1e-2 -- across the capacity buckets and both input sizes; a crop's feature bitwise independent of the batch; features_from_frame
against the reference's slicing; and the drop-in reid_models.OSNet driven through StrongSORT's own call sequence."""
import ctypes as C
import os
import sys

import numpy as np
import pytest

pytestmark = pytest.mark.gpu
torch = pytest.importorskip("torch")

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import osnet_kernel_ref as K  # noqa: E402
from reid_kernel_ref import crop_frame  # noqa: E402
from b200track import _lib as L  # noqa: E402
from oracle import osnet as O  # noqa: E402

DTS = ["fp16", "bf16"]
TDT = {"fp16": torch.float16, "bf16": torch.bfloat16}
SIZES = [(128, 256), (256, 128)]


class TorchMem:
    def put(self, a):
        a = np.ascontiguousarray(a)
        if a.dtype == np.uint16:
            a = a.view(np.int16)
        return torch.from_numpy(a.copy()).cuda()

    def ptr(self, t):
        return C.c_void_p(t.data_ptr())

    def get(self, t):
        torch.cuda.synchronize()
        a = t.cpu().numpy()
        return a.view(np.uint16) if a.dtype == np.int16 else a

    def stream(self):
        return C.c_void_p(torch.cuda.current_stream().cuda_stream)


MEM = TorchMem()


@pytest.fixture(scope="module")
def lib():
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    return L.load()


def geometries(size):
    """(h, w, cin, mid, cout, has a transition) per stage and the head's map, for an input of `size`"""
    H, W = size
    out = []
    h, w = H // 4, W // 4
    for _, cin, cout, trans in O.STAGES:
        out.append((h, w, cin, cout // 4, cout, trans))
        if trans:
            h, w = h // 2, w // 2
    return out, (h, w)


# ---------------------------------------------------------------- kernels against float64

@pytest.mark.parametrize("dt", DTS)
def test_crops_kernel(lib, dt):
    rng = np.random.default_rng(1)
    buf, rows, wins = crop_frame(rng, [(130, 61, 200, 3, 2, 140, 1), (7, 330, 400, 10, 4, 12, 0), (1, 1, 5, 4, 0, 3, 2), (256, 128, 128, 0, 0, 256, 3)])
    for oh, ow in SIZES:
        out = K.run_crops(lib, MEM, buf, rows, oh, ow, dt)
        for i, win in enumerate(wins):
            K.check16(out[i, ..., :3], K.crop_ref(win, oh, ow), K.CROP_S, dt, "crop %d at %dx%d" % (i, oh, ow))
        assert (out[..., 3] == 0).all()


@pytest.mark.parametrize("dt", DTS)
@pytest.mark.parametrize("size", SIZES)
@pytest.mark.parametrize("pitch", [4, 16])
def test_stem_kernel(lib, dt, size, pitch):
    rng = np.random.default_rng(2)
    x = K.round16(rng.normal(0, 1, (3,) + size + (pitch,)), dt)
    x[..., 3:] = K.NAN16                                              # channels past 3 are never read
    wt = K.rand_weights(rng, (147, 16), 147)
    bias = rng.normal(0, 0.1, 16).astype(np.float32)
    got = K.run_stem(lib, MEM, x, wt, bias, dt)
    xw = K.widen16(x, dt)
    ref, s = K.stem_ref(xw[..., :3], wt, bias)
    K.check16(got, ref, s, dt, "stem")


@pytest.mark.parametrize("dt", DTS)
@pytest.mark.parametrize("size", SIZES)
def test_block_kernels_every_stage(lib, dt, size):
    """conv1, the LightConv3x3, the gate-sum, conv3 (+ downsample or identity) and the transition at each stage's map"""
    rng = np.random.default_rng(3)
    blocks, (hh, hw_) = geometries(size)
    n = 2
    W = lambda a: None if a is None else K.widen16(a, dt)        # noqa: E731
    for h, w, cin, mid, cout, trans in blocks:
        for ci in (cin, cout):
            x = K.rand_act(rng, (n, h, w, ci), dt)
            wt = K.rand_weights(rng, (ci, mid), ci)
            b = rng.normal(0, 0.2, mid).astype(np.float32)
            got = K.run_pointwise(lib, MEM, x, None, wt, b, None, True, False, dt)
            ref, s = K.pointwise_ref(W(x), None, wt, b, None, True, False)
            K.check16(got, ref, s, dt, "conv1 %s" % ((h, w, ci, mid),))
            x1 = K.rand_act(rng, (n, h, w, mid), dt)
            w1, dw = K.rand_weights(rng, (mid, mid), mid), K.rand_weights(rng, (9, mid), 9)
            lb = rng.normal(0, 0.2, mid).astype(np.float32)
            got = K.run_lightconv(lib, MEM, x1, w1, dw, lb, dt)
            ref, s = K.lightconv_ref(W(x1), w1, dw, lb)
            K.check16(got, ref, s, dt, "lightconv %s" % ((h, w, mid),))
            streams = [K.rand_act(rng, (n, h * w, mid), dt) for _ in range(4)]
            hid = mid // 16
            fc = (K.rand_weights(rng, (hid, mid), mid, 2.0), rng.normal(0, 0.1, hid).astype(np.float32),
                  K.rand_weights(rng, (mid, hid), hid, 2.0), rng.normal(0, 0.1, mid).astype(np.float32))
            got = K.run_gate(lib, MEM, streams, *fc, dt)
            ref, s, _ = K.gate_ref([W(a) for a in streams], *fc)
            K.check16(got, ref, s, dt, "gate %s" % ((h * w, mid, hid),))
            x2 = K.rand_act(rng, (n, h, w, mid), dt)
            w3 = K.rand_weights(rng, (mid + (ci if ci != cout else 0), cout), mid)
            b3 = rng.normal(0, 0.2, cout).astype(np.float32)
            xb, res = (x, None) if ci != cout else (None, K.rand_act(rng, (n, h, w, cout), dt, relu=False))
            if ci == cout:
                x = res
            got = K.run_pointwise(lib, MEM, x2, xb, w3, b3, res, True, False, dt)
            ref, s = K.pointwise_ref(W(x2), W(xb), w3, b3, W(res), True, False)
            K.check16(got, ref, s, dt, "conv3 %s" % ((h, w, mid, ci, cout),))
        if trans:
            x = K.rand_act(rng, (n, h, w, cout), dt)
            wt = K.rand_weights(rng, (cout, cout), cout)
            b = rng.normal(0, 0.2, cout).astype(np.float32)
            got = K.run_pointwise(lib, MEM, x, None, wt, b, None, True, True, dt)
            ref, s = K.pointwise_ref(W(x), None, wt, b, None, True, True)
            K.check16(got, ref, s, dt, "transition %s" % ((h, w, cout),))
    x = K.rand_act(rng, (n, hh * hw_, 128), dt)
    wt = K.rand_weights(rng, (128, 512), 128)
    b = rng.normal(0, 0.3, 512).astype(np.float32)
    got = K.run_head(lib, MEM, x, wt, b, dt)
    ref, bound = K.head_ref(W(x), wt, b)
    K.assert_bound(got, ref, bound, "head")


def test_pointwise_grid_stride_wraps(lib):
    """more items than the persistent grid covers in one pass (132 * 4 blocks x 256 threads)"""
    rng = np.random.default_rng(4)
    x = K.rand_act(rng, (40, 32, 64, 16), "fp16")
    wt = K.rand_weights(rng, (16, 64), 16)
    b = rng.normal(0, 0.2, 64).astype(np.float32)
    got = K.run_pointwise(lib, MEM, x, None, wt, b, None, True, False, "fp16")
    ref, s = K.pointwise_ref(K.widen16(x, "fp16"), None, wt, b, None, True, False)
    K.check16(got, ref, s, "fp16", "pointwise wrap")


# ---------------------------------------------------------------- the extractor against the fp32 oracle

@pytest.fixture(scope="module")
def sd():
    return O.seeded_state_dict(0)


_EXT = {}


def extractor(sd, size, dt="fp16"):
    from b200track.osnet import OsnetExtractor
    key = (size, dt)
    if key not in _EXT:
        _EXT[key] = OsnetExtractor(sd, device="cuda:0", dtype=TDT[dt], size=size)
    return _EXT[key]


def oracle_feats(sd, x):
    sdc = {k: v.cuda() for k, v in sd.items()}
    with torch.no_grad():
        return torch.cat([O.forward(sdc, x[i:i + 128]) for i in range(0, len(x), 128)])


def assert_parity(f, ref, what):
    f, ref = f.double(), ref.double()
    cos = (f * ref).sum(1) / (f.norm(dim=1) * ref.norm(dim=1))
    rel = (f - ref).norm(dim=1) / ref.norm(dim=1)
    assert float(cos.min()) >= 0.9999 and float(rel.max()) <= 1e-2, "%s: min cosine %.6f, max relative L2 %.2e" % (what, cos.min(), rel.max())
    print("%s: min cosine %.7f, max relative L2 %.2e" % (what, float(cos.min()), float(rel.max())))


def frames_and_boxes(seed, n, fh=360, fw=640):
    rng = np.random.default_rng(seed)
    frame = np.ascontiguousarray(np.clip(rng.normal(128, 60, (fh // 8 + 1, fw // 8 + 1, 3)).repeat(8, 0).repeat(8, 1)[:fh, :fw]
                                         + rng.normal(0, 10, (fh, fw, 3)), 0, 255).astype(np.uint8))
    x1 = rng.uniform(0, fw - 4, n); y1 = rng.uniform(0, fh - 4, n)
    bw = rng.uniform(2, 200, n); bh = rng.uniform(2, 300, n)
    boxes = np.stack([x1, y1, x1 + bw, y1 + bh], 1)                   # right / bottom ends may pass the frame: the slice clips them
    boxes[0] = [0, 0, fw + 30.7, fh + 12.2]
    if n > 1:
        boxes[1] = [fw - 1.5, fh - 2.5, fw + 5, fh + 5]
    return frame, boxes


def reference_crops(frame, boxes):
    """StrongSORT.get_feature's slicing: tlbr = list(map(int, tlbr)); ori_img[y1:y2, x1:x2]"""
    out = []
    for b in boxes:
        x1, y1, x2, y2 = [int(v) for v in b]
        out.append(frame[y1:y2, x1:x2])
    return out


@pytest.mark.parametrize("size", SIZES)
def test_extractor_against_oracle(lib, sd, size):
    ext = extractor(sd, size)
    frame, boxes = frames_and_boxes(5, 1000)
    x = O.preprocess(reference_crops(frame, boxes), size).cuda()
    ref = oracle_feats(sd, x)
    d_frame = torch.from_numpy(frame).cuda()
    for n in (1, 31, 32, 33, 256, 1000):
        f = ext.features_from_frame(d_frame, boxes[:n])
        assert f.shape == (n, 512) and f.dtype == torch.float32
        assert_parity(f, ref[:n], "features_from_frame %s n=%d" % (size, n))
        g = ext.forward_nchw(x[:n])
        assert_parity(g, ref[:n], "forward_nchw %s n=%d" % (size, n))


def test_extractor_bf16_against_oracle(lib, sd):
    ext = extractor(sd, (128, 256), "bf16")
    frame, boxes = frames_and_boxes(6, 64)
    ref = oracle_feats(sd, O.preprocess(reference_crops(frame, boxes)).cuda())
    f = ext.features_from_frame(frame, boxes).double()
    cos = (f * ref.double()).sum(1) / (f.norm(dim=1) * ref.double().norm(dim=1))
    assert float(cos.min()) >= 0.999, float(cos.min())              # bf16 keeps 3 fewer mantissa bits than fp16


def test_feature_independent_of_batch(lib, sd):
    ext = extractor(sd, (128, 256))
    frame, boxes = frames_and_boxes(7, 300)
    d = torch.from_numpy(frame).cuda()
    alone = ext.features_from_frame(d, boxes[:5]).clone()
    net = ext.last_net
    net["x4"][5:].view(torch.int16).fill_(-1)                         # NaN in the padding rows of the bucket
    again = ext.features_from_frame(d, boxes[:5]).clone()
    assert torch.equal(alone, again)
    for n in (33, 300):                                               # other buckets, other positions
        order = np.random.default_rng(n).permutation(n)
        big = ext.features_from_frame(d, boxes[order])
        pos = [int(np.flatnonzero(order == i)[0]) for i in range(5)]
        assert torch.equal(big[pos], alone), "a crop's feature changed with n = %d / its position" % n


def test_features_from_frame_edges_and_errors(lib, sd):
    ext = extractor(sd, (128, 256))
    frame, _ = frames_and_boxes(8, 2)
    fh, fw = frame.shape[:2]
    boxes = np.array([[0, 0, 5, 7], [fw - 3, fh - 9, fw + 100, fh + 100], [10.9, 20.99, 11.01, 21.5], [0.4, 0.6, fw, fh]])
    f = ext.features_from_frame(frame, boxes)
    ref = oracle_feats(sd, O.preprocess(reference_crops(frame, boxes)).cuda())
    assert_parity(f, ref, "edge boxes")
    assert ext.features_from_frame(frame, np.zeros((0, 4))).shape == (0, 512)
    with pytest.raises(L.B2TError, match="negative"):
        ext.features_from_frame(frame, [[-1.5, 0, 10, 10]])
    with pytest.raises(L.B2TError, match="empty"):
        ext.features_from_frame(frame, [[5, 5, 5.9, 20]])
    with pytest.raises(L.B2TError, match="empty"):
        ext.features_from_frame(frame, [[fw + 1, 0, fw + 20, 10]])


def test_extractor_argument_errors(lib, sd):
    from b200track.osnet import OsnetExtractor
    with pytest.raises(L.B2TError, match="multiples of 16"):
        OsnetExtractor(sd, size=(100, 256))
    bad = dict(sd)
    bad.pop("conv2.0.gate.fc1.weight")
    with pytest.raises(L.B2TError, match="lacks"):
        OsnetExtractor(bad)
    ext = extractor(sd, (128, 256))
    with pytest.raises(L.B2TError, match="built for"):
        ext.forward_nchw(torch.zeros((1, 3, 256, 128), device="cuda"))
    with pytest.raises(L.B2TError, match="float32"):
        ext.forward_nchw(torch.zeros((1, 3, 128, 256), device="cuda", dtype=torch.float16))
    with pytest.raises(L.B2TError):
        OsnetExtractor(sd, dtype=torch.float32)


# ---------------------------------------------------------------- the drop-in module, driven as strongsort.py drives it

def test_dropin_through_strongsort_call_sequence(lib, sd, tmp_path):
    sys.path.insert(0, os.path.join(os.path.dirname(HERE), "yolov7-tracker_b200", "tracker"))
    try:
        from reid_models.OSNet import osnet_x0_25
    finally:
        sys.path.pop(0)
        for k in [k for k in sys.modules if k == "reid_models" or k.startswith("reid_models.")]:
            sys.modules.pop(k)
    # strongsort.py:26-29: construct, .cuda().eval(), load_pretrained_weights(model, path) -- restated: torch.load, strip "module.",
    # keep the tensors whose name and shape match, model_dict.update, load_state_dict
    model = osnet_x0_25(num_classes=1, pretrained=False)
    model.cuda().eval()
    ck = {"module." + k: v for k, v in sd.items() if not k.startswith("classifier")}
    ck["module.classifier.weight"] = torch.randn(1041, 512)
    path = tmp_path / "osnet_x0_25.pth"
    torch.save(ck, path)
    state_dict = torch.load(path, map_location="cuda")
    model_dict = model.state_dict()
    new = {}
    for k, v in state_dict.items():
        k = k[7:] if k.startswith("module.") else k
        if k in model_dict and model_dict[k].size() == v.size():
            new[k] = v
    assert len(new) == 565
    model_dict.update(new)
    model.load_state_dict(model_dict)
    # get_feature :66-89: a stack of preprocessed crops, .cuda(), model(x).cpu().detach().numpy()
    frame, boxes = frames_and_boxes(9, 20)
    x = O.preprocess(reference_crops(frame, boxes))
    feats = model(x.cuda()).cpu().detach().numpy()
    assert feats.shape == (20, 512) and feats.dtype == np.float32
    ref = oracle_feats(sd, x.cuda())
    assert_parity(torch.from_numpy(feats).cuda(), ref, "drop-in")
    # weights loaded after a forward are used by the next one
    sd2 = dict(sd)                                                    # other weights, same conditioning: the fc rows permuted
    perm = torch.from_numpy(np.random.default_rng(3).permutation(512))
    for k in ("fc.0.weight", "fc.0.bias", "fc.1.weight", "fc.1.bias", "fc.1.running_mean", "fc.1.running_var"):
        sd2[k] = sd[k][perm].clone()
    model.load_state_dict(sd2)
    assert_parity(model(x.cuda()), oracle_feats(sd2, x.cuda()), "drop-in after reload")
    with pytest.raises(RuntimeError):
        model.train()(x.cuda())
    with pytest.raises(RuntimeError, match="CUDA"):
        model.eval()(x)
