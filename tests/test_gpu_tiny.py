"""-m gpu: YOLOv7-tiny (BASELINE.json configs[0]: cfg/deploy/yolov7-tiny.yaml -- LeakyReLU convs, MP / SP pools, three Detect levels)
on the GPU kernels against oracle/detector.py, which tests/test_oracle_detector.py pins against the reference's own Model."""
import pytest

pytestmark = pytest.mark.gpu
torch = pytest.importorskip("torch")


@pytest.mark.parametrize("shape,autotune", [((256, 320), False), ((640, 640), True)])
def test_detector_tiny_end_to_end_vs_oracle(shape, autotune):
    from b200track import tiny
    from oracle import detector as OD
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    sd = tiny.seeded_state_dict(0)
    img = torch.rand((2, 3) + shape, generator=torch.Generator().manual_seed(11)).cuda()
    det = tiny.DetectorTiny(sd, batch=2, img_size=shape, use_graph=False, autotune=autotune)
    pred = det.forward(img).clone()
    torch.cuda.synchronize()
    sd_gpu = {k: v.cuda() for k, v in sd.items()}
    L_ = tiny.tiny_layers()
    with torch.no_grad():
        ref16, raw16 = OD.forward(L_, sd_gpu, img, tiny.ANCHORS, tiny.STRIDES, emulate_bf16=det.act_dtype, return_raw=True, act="leaky", name_offset=-1)
        ref32 = OD.forward(L_, sd_gpu, img, tiny.ANCHORS, tiny.STRIDES, act="leaky", name_offset=-1)
    assert pred.shape == ref32.shape
    for lvl, r in enumerate(raw16):                                  # raw logits vs the oracle with the same 16-bit rounding
        got = det.raw[lvl][..., :255].reshape(2, r.shape[2], r.shape[3], 3, 85).permute(0, 3, 1, 2, 4)
        err = (got - r).abs()
        assert float(err.max()) < 0.05 and float(err.mean()) < 3e-3, "level %d: max %.3f mean %.4f" % (lvl, err.max(), err.mean())
    d32 = (pred - ref32).abs()
    print("tiny %s: max |d obj| vs fp32 oracle %.2e, mean %.2e" % (shape, float(d32[..., 4].max()), float(d32[..., 4].mean())))
    assert float(d32[..., 4].max()) < 5e-3                           # objectness against exact fp32
    rel = d32[..., :4] / (ref32[..., :4].abs() + 1.0)
    assert float(rel.max()) < 0.05 and float(rel.mean()) < 2e-3
    out, cnt = det.detect(img, post=False)
    torch.cuda.synchronize()
    ref_nms = OD.non_max_suppression(pred, conf_thres=0.01)          # same pred -> the NMS must agree exactly
    for b in range(2):
        n = int(cnt[b])
        assert n > 0 and n == ref_nms[b].shape[0] and torch.equal(out[b, :n, 5], ref_nms[b][:, 5])
        assert torch.allclose(out[b, :n, :5], ref_nms[b][:, :5], atol=1e-3)


def test_tiny_refuses_uint8_ingest():
    from b200track import _lib as L
    from b200track import tiny
    det = tiny.DetectorTiny(tiny.seeded_state_dict(0), batch=1, img_size=128, use_graph=False, autotune=False)
    with pytest.raises(L.B2TError):
        det.set_source_frames((128, 128))


def test_dropin_model_runs_the_tiny_graph():
    """models.yolo.Model('cfg/deploy/yolov7-tiny.yaml') -- the reference's constructor call -- on the drop-in: stride 32, model(img)[0]
    equal to the engine's prediction, raw maps in the reference's (B, na, ny, nx, no) layout."""
    import os
    import sys
    root = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "yolov7-tracker_b200")
    sys.path.insert(0, root)
    try:
        for k in [k for k in sys.modules if k == "models" or k.startswith("models.")]:
            del sys.modules[k]
        from models.yolo import Model
    finally:
        sys.path.remove(root)
    from b200track import tiny
    from oracle import detector as OD
    sd = tiny.seeded_state_dict(2)
    m = Model("cfg/deploy/yolov7-tiny.yaml").load_state_dict(sd)
    assert int(m.stride.max()) == 32
    img = torch.rand((1, 3, 160, 224), generator=torch.Generator().manual_seed(3)).cuda()
    pred, raw = m(img)
    with torch.no_grad():
        ref = OD.forward(tiny.tiny_layers(), {k: v.cuda() for k, v in sd.items()}, img, tiny.ANCHORS, tiny.STRIDES, act="leaky", name_offset=-1)
    assert pred.shape == ref.shape and float((pred[..., 4] - ref[..., 4]).abs().max()) < 5e-3
    assert [tuple(r.shape) for r in raw] == [(1, 3, 20, 28, 85), (1, 3, 10, 14, 85), (1, 3, 5, 7, 85)]
    with pytest.raises(ValueError):
        m(torch.zeros((1, 3, 100, 224)).cuda())
