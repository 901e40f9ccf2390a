"""-m gpu: the NMS stage (csrc/b2t_nms.cu) on the nvcc build at the edges where it can go wrong, bit for bit against the float32
restatement of tests/nms_ref.py: threshold confidences and IoUs (exactly at the fp32 threshold and one ulp either side), ties at
1.0 through the max_nms cut, confidences above 1, zero-area boxes, class-offset boxes across 4096, block edges of the greedy scan
(max_det 1 / 63 / 64 / 65 / 2048), empty images inside a batch of 8; the fused decode + NMS against decode then NMS; the post
geometry (scale_coords back to a letterboxed source frame) against torch's own arithmetic on the device and the float64 band;
and the refusal of a candidate buffer smaller than the rows per image."""
import ctypes as C
import os
import sys

import numpy as np
import pytest

pytestmark = pytest.mark.gpu
torch = pytest.importorskip("torch")

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import nms_ref as R  # noqa: E402
from b200track import _lib as L  # noqa: E402


@pytest.fixture(scope="module")
def lib():
    return L.load()


def _s():
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def _nms(lib, pred, conf, iou, max_det, max_nms, post=0, geo=(1.0, 0.0, 0.0), img=(640.0, 640.0), max_cand=None):
    """pred: (B, N, no) float32 CUDA tensor -> (rc, out, count) of b2t_nms"""
    B, N, no = pred.shape
    max_cand = N if max_cand is None else max_cand
    ws = torch.empty(max(1, lib.b2t_nms_workspace_bytes(B, max(max_cand, 1), max_nms)), dtype=torch.uint8, device="cuda")
    out = torch.full((B, max_det, 6), -7.0, device="cuda"); cnt = torch.full((B,), -1, dtype=torch.int32, device="cuda")
    rc = lib.b2t_nms(C.c_void_p(pred.data_ptr()), B, N, no, conf, iou, max_det, max_nms, max_cand, post, *geo, img[0], img[1],
                     C.c_void_p(ws.data_ptr()), ws.numel(), C.c_void_p(out.data_ptr()), C.c_void_p(cnt.data_ptr()), _s())
    torch.cuda.synchronize()
    return rc, out, cnt


def _check_bits(out, cnt, ref, what):
    out, cnt = out.cpu().numpy(), cnt.cpu().numpy()
    for b, r in enumerate(ref):
        n = int(cnt[b])
        bad = R.first_row_mismatch(out[b, :n], r["rows"])
        assert bad is None, "%s image %d: first differing row %d (%d rows, expected %d)" % (what, b, bad, n, len(r["rows"]))
        # every decision where float64 would decide otherwise lies within rounding of the threshold
        assert all(m < R.IOU_BAND for _, k32, k64, m in r["decisions"] if k32 != k64), what


@pytest.mark.parametrize("name", sorted(R.edge_cases(large=True)))
def test_b2t_nms_edge_cases_bit_equal_nms_ref(lib, name):
    pred, conf, iou, max_det, max_nms = R.edge_cases(large=True)[name]
    rc, out, cnt = _nms(lib, torch.from_numpy(pred).cuda(), conf, iou, max_det, max_nms)
    assert rc == 0, lib.b2t_detect_last_error()
    ref = R.nms_ref(pred, conf, iou, max_det, max_nms)
    _check_bits(out, cnt, ref, name)
    if name.startswith("ties_102000"):
        assert list(ref[0]["ranked"]) == list(range(30000))          # the max_nms cut keeps the lowest 30 000 row indices


_BATCH = {}


@pytest.mark.parametrize("conf", [0.0, 0.01, 0.25, 0.999])
@pytest.mark.parametrize("iou", [0.0, 0.45, 1.0])
@pytest.mark.parametrize("max_det", [1, 63, 64, 65, 300, 2048])
def test_b2t_nms_batch_of_edge_sizes_bit_equal_nms_ref(lib, max_det, iou, conf):
    """B = 8 images of 0, 1, 63, 64, 65, ~5 000, 64 and 1 candidates"""
    if "p" not in _BATCH:
        _BATCH["p"] = R.batch_pred()
        _BATCH["t"] = torch.from_numpy(_BATCH["p"]).cuda()
    rc, out, cnt = _nms(lib, _BATCH["t"], conf, iou, max_det, 30000)
    assert rc == 0, lib.b2t_detect_last_error()
    _check_bits(out, cnt, R.nms_ref(_BATCH["p"], conf, iou, max_det, 30000), "max_det %d iou %g conf %g" % (max_det, iou, conf))


# ---------------------------------------------------------------- fused decode + NMS == decode, then NMS

def _head_levels(B, no, seed):
    g = torch.Generator().manual_seed(seed)
    levels = [(16, 12, 8.0, [12, 16, 19, 36, 40, 28]), (8, 6, 16.0, [36, 75, 76, 55, 72, 146]), (4, 3, 32.0, [142, 110, 192, 243, 459, 401])]
    pitch = 3 * no + 5
    raws, arr, off = [], (L.HeadLevel * len(levels))(), 0
    for k, (h, w, stride, anc) in enumerate(levels):
        raw = torch.randn((B, h, w, pitch), generator=g) * 2.0
        raws.append(raw.cuda())
        arr[k].raw = raws[k].data_ptr(); arr[k].raw_pitch = pitch; arr[k].h = h; arr[k].w = w; arr[k].stride = stride
        for j in range(6):
            arr[k].anchors[j] = float(anc[j])
        arr[k].level_off = off
        off += 3 * h * w
    return raws, arr, levels, pitch, off


def test_detect_nms_fused_equals_decode_then_nms_at_threshold_confidences(lib):
    """raw head maps decoded by b2t_detect_decode; the thresholds are then set to confidences that rows of that `pred` hold
    exactly (sigmoid(obj) * sigmoid(cls) on the device), so rows sit at the threshold: the fused path must give the same rows as
    decode -> b2t_nms, and both the rows of nms_ref on that pred"""
    B, no = 3, 9
    raws, arr, levels, pitch, N = _head_levels(B, no, 7)
    pred = torch.zeros((B, N, no), device="cuda")
    for k, (h, w, stride, anc) in enumerate(levels):
        a = (C.c_float * 6)(*[float(v) for v in anc])
        assert lib.b2t_detect_decode(C.c_void_p(raws[k].data_ptr()), pitch, C.c_void_p(pred.data_ptr()), B, h, w, 3, no, arr[k].level_off, N,
                                     float(stride), a, _s()) == 0
    torch.cuda.synchronize()
    p = pred.cpu().numpy()
    conf_rows = (p[..., 5:] * p[..., 4:5]).max(-1)
    qs = np.quantile(conf_rows[0], [0.5, 0.9, 0.99])
    for q in qs:
        thr = float(conf_rows[0].flat[np.argmin(np.abs(conf_rows[0] - q))])     # a confidence some row has exactly
        for iou in (0.45, 0.0):
            rc, out2, cnt2 = _nms(lib, pred, thr, iou, 300, 30000)
            assert rc == 0
            ws = torch.empty(lib.b2t_nms_workspace_bytes(B, N, 30000), dtype=torch.uint8, device="cuda")
            out = torch.zeros((B, 300, 6), device="cuda"); cnt = torch.zeros(B, dtype=torch.int32, device="cuda")
            assert lib.b2t_detect_nms(C.cast(arr, C.c_void_p), len(levels), B, no, thr, iou, 300, 30000, N, 0, 1.0, 0.0, 0.0, 1.0, 1.0,
                                      C.c_void_p(ws.data_ptr()), ws.numel(), C.c_void_p(out.data_ptr()), C.c_void_p(cnt.data_ptr()), _s()) == 0
            torch.cuda.synchronize()
            assert torch.equal(cnt, cnt2)
            for b in range(B):
                n = int(cnt[b])
                assert torch.equal(out[b, :n], out2[b, :n]), "thr %r iou %g image %d" % (thr, iou, b)
            _check_bits(out, cnt, R.nms_ref(p, thr, iou, 300, 30000), "fused thr %r" % thr)


def test_w6_bench_configuration_rows_equal_nms_ref_on_own_pred():
    """the w6 at 1280 x 1280, batch 8, calibrated weights, autotuned, CUDA graph: detect(post=False) == nms_ref on the kernel's own
    pred (decode of the same head maps), and == the two-step decode -> b2t_nms, bit for bit"""
    from b200track.detector import DetectorW6
    from b200track.w6 import calibrated_state_dict
    sd = calibrated_state_dict(0, 1280, "cuda")
    det = DetectorW6(sd, batch=8, img_size=1280, use_graph=True, autotune=True)
    img = torch.rand((8, 3, 1280, 1280), generator=torch.Generator(device="cuda").manual_seed(4), device="cuda")
    out, cnt = det.detect(img, post=False)
    torch.cuda.synchronize()
    out, cnt = out.clone(), cnt.clone()
    pred = det.decode().cpu().numpy()                                # the head maps of the same forward
    out2, cnt2 = det.nms_from_pred(post=False)
    torch.cuda.synchronize()
    assert torch.equal(cnt, cnt2)
    ref = R.nms_ref(pred, det.conf_thres, det.iou_thres, det.max_det, det.max_nms)
    _check_bits(out, cnt, ref, "w6 1280 batch 8")
    for b in range(8):
        assert torch.equal(out[b, :int(cnt[b])], out2[b, :int(cnt[b])])
    assert int(cnt.sum()) > 8


# ---------------------------------------------------------------- post geometry: scale_coords back to the source frame

@pytest.mark.parametrize("k", range(len(R.GEOMETRIES)))
def test_post_geometry_equals_torch_scale_coords_on_device(lib, k):
    """b2t_nms(post=1, gain, pad, source size) == the drop-in scale_coords(canvas, rows_post0, src).round() run on CUDA tensors
    (tracker/track.py:240 on the device), exactly; and inside the float64 band of scale_coords_ref"""
    from b200track.preprocess import scale_coords_geometry
    from utils.general import scale_coords
    src, canvas = R.GEOMETRIES[k]
    rows = np.load(os.path.join(HERE, "golden", "scale_coords.npz"))["rows%d" % k]
    n = len(rows)
    pred = np.zeros((1, n, 6), np.float32)
    pred[0, :, 0] = (rows[:, 0] + rows[:, 2]) / 2; pred[0, :, 2] = rows[:, 2] - rows[:, 0]
    pred[0, :, 1] = (rows[:, 1] + rows[:, 3]) / 2; pred[0, :, 3] = rows[:, 3] - rows[:, 1]
    pred[0, :, 4] = np.linspace(0.99, 0.5, n, dtype=np.float32)
    pred[0, :, 5] = 1.0
    t = torch.from_numpy(pred).cuda()
    geo = scale_coords_geometry(canvas, src)
    rc0, post0, c0 = _nms(lib, t, 0.01, 1.0, 300, 30000)
    rc1, post1, c1 = _nms(lib, t, 0.01, 1.0, 300, 30000, post=1, geo=geo, img=(float(src[1]), float(src[0])))
    assert rc0 == rc1 == 0 and int(c0[0]) == int(c1[0]) == n
    exp = post0[0, :n].clone()
    exp[:, :4] = scale_coords(canvas, exp[:, :4], src).round()
    got = post1[0, :n]
    diff = int((got != exp).sum())
    assert diff == 0, "%d coordinates differ from torch's scale_coords on the device" % diff
    lo, hi, _ = R.scale_coords_ref(post0[0, :n].cpu().numpy(), canvas, src)
    assert len(R.outside_band(got.cpu().numpy(), lo, hi)) == 0
    cpu = post0[0, :n].cpu().clone()
    cpu[:, :4] = scale_coords(canvas, cpu[:, :4], src).round()
    print("\n%s -> %s: CPU torch differs from CUDA torch on %d coordinates" % (src, canvas, int((cpu != got.cpu()).sum())))


def test_max_cand_below_rows_per_image_refused(lib):
    pred = torch.zeros((2, 100, 8), device="cuda")
    rc, _, _ = _nms(lib, pred, 0.01, 0.45, 10, 100, max_cand=99)
    assert rc == -1                                                  # B2T_EINVAL
    assert b"max_cand" in lib.b2t_detect_last_error()
    raws, arr, levels, pitch, N = _head_levels(2, 8, 1)
    ws = torch.empty(lib.b2t_nms_workspace_bytes(2, N, N), dtype=torch.uint8, device="cuda")
    out = torch.zeros((2, 10, 6), device="cuda"); cnt = torch.zeros(2, dtype=torch.int32, device="cuda")
    for mc, want in ((N - 1, -1), (N, 0)):
        rc = lib.b2t_detect_nms(C.cast(arr, C.c_void_p), len(levels), 2, 8, 0.01, 0.45, 10, N, mc, 0, 1.0, 0.0, 0.0, 1.0, 1.0,
                                C.c_void_p(ws.data_ptr()), ws.numel(), C.c_void_p(out.data_ptr()), C.c_void_p(cnt.data_ptr()), _s())
        assert rc == want, (mc, lib.b2t_detect_last_error())
    torch.cuda.synchronize()
