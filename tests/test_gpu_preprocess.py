"""-m gpu: b2t_letterbox (csrc/b2t_preproc.cu) on the nvcc build, through b200track.preprocess.Letterbox: bit-exact against
the committed outputs of the reference's own pre-processing (tracker/tracker_dataloader.py:64-130) and against the oracle at
the full 1080p -> 1280 size of BASELINE's frames.  Integer resize arithmetic + IEEE float / 255: tolerance 0."""
import os

import numpy as np
import pytest

pytestmark = pytest.mark.gpu
torch = pytest.importorskip("torch")

GOLDEN = os.path.join(os.path.dirname(__file__), "golden", "letterbox.npz")


def test_letterbox_matches_reference_golden():
    from b200track.preprocess import Letterbox
    g = np.load(GOLDEN)
    for k, (h, w, size, stride) in enumerate(g["cases"]):
        out, geo = Letterbox(int(size), int(stride))(g["img%d" % k])
        torch.cuda.synchronize()
        ref = g["out%d" % k]
        assert tuple(out.shape[1:]) == ref.shape
        assert np.array_equal(out[0].cpu().numpy(), ref), "case %d: %d values differ" % (k, int((out[0].cpu().numpy() != ref).sum()))


def test_letterbox_1080p_batch_matches_oracle():
    from b200track.preprocess import Letterbox
    from oracle import preprocess as P
    rng = np.random.default_rng(5)
    frames = rng.integers(0, 256, (2, 1080, 1920, 3), dtype=np.uint8)
    lb = Letterbox(1280, 64)
    out, geo = lb(torch.from_numpy(frames).cuda())                  # device-resident uint8 input
    torch.cuda.synchronize()
    assert tuple(out.shape) == (2, 3, 768, 1280) and (geo["top"], geo["left"]) == (24, 0)
    for b in range(2):
        ref, _ = P.preprocess(frames[b], (1280, 1280), 64)
        assert np.array_equal(out[b].cpu().numpy(), ref)
    out2, _ = lb(frames)                                            # host frames through pinned memory: same result
    torch.cuda.synchronize()
    assert torch.equal(out, out2)


def test_letterboxed_frame_through_non_square_detector():
    """uint8 frame -> b2t_letterbox (stride 128 so that both sides suit ReOrg + stride 64) -> DetectorW6 on the resulting
    384 x 512 rectangle: logits against the bf16-emulating oracle (statistically, like the 640 x 640 test), decode + NMS exactly."""
    from b200track.detector import DetectorW6
    from b200track.preprocess import Letterbox
    from b200track.w6 import ANCHORS, STRIDES, calibrated_state_dict, w6_layers
    from oracle import detector as OD
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    rng = np.random.default_rng(11)
    frame = rng.integers(0, 256, (270, 480, 3), dtype=np.uint8)
    img, geo = Letterbox(512, 128)(frame)
    assert tuple(img.shape) == (1, 3, 384, 512) and (geo["top"], geo["left"]) == (48, 0)
    sd = calibrated_state_dict(0, 512, "cuda", img=img)             # LSUV pass on THIS canvas (gray borders): the 300-row cap is hit
    det = DetectorW6(sd, batch=1, img_size=(384, 512), use_graph=False)
    pred = det.forward(img).clone()
    out, cnt = det.detect(img, post=True)
    torch.cuda.synchronize()
    with torch.no_grad():
        ref_bf, raw_bf = OD.forward(w6_layers(), sd, img, ANCHORS, STRIDES, emulate_bf16=det.act_dtype, return_raw=True)
    assert tuple(pred.shape) == tuple(ref_bf.shape)
    for lvl, r in enumerate(raw_bf):
        got = det.raw[lvl][..., :255].reshape(1, r.shape[2], r.shape[3], 3, 85).permute(0, 3, 1, 2, 4)
        err = (got - r).abs()
        rel_rms = float((err ** 2).mean().sqrt() / r.std())
        assert float(err.mean()) < 0.12 and rel_rms < 0.12, "level %d: mean %.4f rel rms %.3f" % (lvl, err.mean(), rel_rms)
    ref = OD.post_process(OD.non_max_suppression(pred, conf_thres=0.01)[0], (384, 512))
    n = int(cnt[0])
    assert n == ref.shape[0] and n > 0
    assert torch.equal(out[0, :n, 5], ref[:, 5]) and torch.allclose(out[0, :n, :5], ref[:, :5], atol=1e-3)
    assert float(out[0, :n, 2].max()) <= 512 and float(out[0, :n, 3].max()) <= 384      # clipped to (W, H)


@pytest.mark.parametrize("act", ["fp16", "bf16"])
def test_letterbox_reorg_fused_on_gpu_equals_two_steps_and_oracle(act):
    """b2t_letterbox_reorg on the GPU (uint8 BGR frames -> the detector's padded ReOrg / NHWC 16-bit input, one kernel) ==
    b2t_letterbox (float canvas, already pinned bit-exact against the reference's own output) followed by b2t_image_reorg_padded,
    bit for bit, for a resized 1080p frame pair and a same-size frame; and == the oracle's canvas pushed through ReOrg + torch's
    rounding.  Integer resize arithmetic + IEEE division + round-to-nearest-even conversion: tolerance 0."""
    import ctypes as C
    from b200track import _lib as L
    from b200track.preprocess import Letterbox, launch_letterbox_reorg, letterbox_geometry
    from oracle import preprocess as P
    lib = L.load()
    dt = torch.float16 if act == "fp16" else torch.bfloat16
    code = L.act_dtype_code(dt)
    rng = np.random.default_rng(21)
    for (h, w, size) in ((1080, 1920, 1280), (256, 256, 256), (270, 480, 512)):
        frames = rng.integers(0, 256, (2, h, w, 3), dtype=np.uint8)
        u8 = torch.from_numpy(frames).cuda()
        canvas, geo = Letterbox(size, 64)(u8)
        H2, W2 = geo["out_h"] // 2, geo["out_w"] // 2
        row = W2 + 8
        two = torch.full((2, H2, row, 16), 3.0, dtype=dt, device="cuda")
        s = C.c_void_p(torch.cuda.current_stream().cuda_stream)
        assert lib.b2t_image_reorg_padded(C.c_void_p(canvas.data_ptr()), C.c_void_p(two.data_ptr()), 2, geo["out_h"], geo["out_w"], row, 1, code, s) == 0
        one = torch.full((2, H2, row, 16), 3.0, dtype=dt, device="cuda")
        launch_letterbox_reorg(lib, u8.data_ptr(), 2, h, w, 3 * w, geo, one.data_ptr(), row, 1, s, act_dtype=code)
        torch.cuda.synchronize()
        assert torch.equal(one.view(torch.int16), two.view(torch.int16)), (h, w, size)
        ref, _ = P.preprocess(frames[1], (size, size), 64)                      # oracle canvas (3, H, W) float32
        x = torch.from_numpy(ref)[None]
        re = torch.cat([x[..., ::2, ::2], x[..., 1::2, ::2], x[..., ::2, 1::2], x[..., 1::2, 1::2]], 1)[0].permute(1, 2, 0).to(dt)
        assert torch.equal(one[1, :, 1:W2 + 1, :12].cpu().view(torch.int16), re.contiguous().view(torch.int16))
        assert bool((one[:, :, 0] == 3.0).all()) and bool((one[:, :, W2 + 1:] == 3.0).all()) and bool((one[:, :, 1:W2 + 1, 12:] == 0).all())


def test_pipeline_uint8_frames_equal_float_frames():
    """TrackingPipeline fed uint8 BGR frames (device-side letterbox + ReOrg, 3 bytes per pixel over PCIe) returns the same track
    rows, frame by frame, as the pipeline fed the float tensors the reference's dataloader would produce from those frames."""
    from b200track import _lib as L
    from b200track.detector import DetectorW6
    from b200track.engine import TrackEngine
    from b200track.pipeline import TrackingPipeline
    from b200track.w6 import calibrated_state_dict
    sd = calibrated_state_dict(0, 256, "cuda")
    rng = np.random.default_rng(33)
    base = rng.integers(0, 256, (2, 256, 256, 3), dtype=np.uint8)
    frames_u8 = [torch.from_numpy(np.roll(base, (2 * k, k), axis=(1, 2)).copy()).pin_memory() for k in range(5)]
    frames_f = [(f.flip(-1).permute(0, 3, 1, 2).float() / 255.0).contiguous().pin_memory() for f in frames_u8]   # BGR->RGB, CHW, /255 (:80-86)
    results = []
    for frames in (frames_u8, frames_f):
        det = DetectorW6(sd, batch=2, img_size=256, use_graph=False, autotune=False)
        if frames is frames_u8:
            geo = det.set_source_frames((256, 256))
            assert (geo["top"], geo["left"], geo["unpad_w"]) == (0, 0, 256)
        eng = TrackEngine("bytetrack", n_seq=2, cap=512, dmax=300)
        pipe = TrackingPipeline(det, eng, out_rows=512)
        got = []
        for f in frames:
            r = pipe.step(f)
            if r is not None:
                got.append([r[0][s, :int(r[1][s, L.STAT_NOUT])].clone() for s in range(2)])
        r = pipe.flush()
        got.append([r[0][s, :int(r[1][s, L.STAT_NOUT])].clone() for s in range(2)])
        results.append(got)
    assert len(results[0]) == len(results[1]) == 5
    n_rows = 0
    for a, b in zip(*results):
        for s in range(2):
            # (a zero-width detection gives a NaN Kalman state in the reference too -- q9 -- so rows may hold NaN: compare with equal_nan)
            assert a[s].shape == b[s].shape and torch.allclose(a[s], b[s], rtol=0, atol=0, equal_nan=True)
            n_rows += a[s].shape[0]
    assert n_rows > 0
    with pytest.raises(L.B2TError):                                              # mismatched engine layout is refused up front
        TrackingPipeline(det, TrackEngine("bytetrack", n_seq=2, cap=512, dmax=256), out_rows=512)


def test_pipeline_twin_detectors_equal_single_detector():
    """TrackingPipeline over two twin detectors (frames alternate; ingest / NMS / association of neighbouring frames overlap the
    forward) returns, frame by frame, exactly the rows of the single-detector pipeline."""
    from b200track import _lib as L
    from b200track.detector import DetectorW6
    from b200track.engine import TrackEngine
    from b200track.pipeline import TrackingPipeline
    from b200track.w6 import calibrated_state_dict
    sd = calibrated_state_dict(0, 256, "cuda")
    rng = np.random.default_rng(34)
    base = rng.integers(0, 256, (2, 256, 256, 3), dtype=np.uint8)
    frames = [torch.from_numpy(np.roll(base, (2 * k, k), axis=(1, 2)).copy()).pin_memory() for k in range(7)]
    results = []
    for n_det in (1, 2):
        dets = []
        for _ in range(n_det):
            d = DetectorW6(sd, batch=2, img_size=256, use_graph=False, autotune=False)
            d.set_source_frames((256, 256))
            dets.append(d)
        pipe = TrackingPipeline(dets if n_det == 2 else dets[0], TrackEngine("bytetrack", n_seq=2, cap=512, dmax=300), out_rows=512)
        got = []
        for f in frames:
            r = pipe.step(f)
            if r is not None:
                got.append([r[0][s, :int(r[1][s, L.STAT_NOUT])].clone() for s in range(2)])
        r = pipe.flush()
        got.append([r[0][s, :int(r[1][s, L.STAT_NOUT])].clone() for s in range(2)])
        results.append(got)
    assert len(results[0]) == len(results[1]) == 7
    rows = 0
    for a, b in zip(*results):
        for s in range(2):
            assert a[s].shape == b[s].shape and torch.allclose(a[s], b[s], rtol=0, atol=0, equal_nan=True)
            rows += a[s].shape[0]
    assert rows > 0
