"""not-gpu: LOGIC of csrc/b2t_nms.cu (filter, counting sort by confidence bins, lazy greedy suppression, fused
Detect decode) executed by the fiber simulator against the oracle's restatement of utils/general.py:607-695.
The `-m gpu` tests repeat this on the nvcc build (tests/test_gpu_detector.py)."""
import ctypes as C
import os
import sys

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.join(os.path.dirname(__file__), "hostsim"))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import nms_ref as R  # noqa: E402
from simlib import ptr, sim  # noqa: E402
from b200track import _lib as L  # noqa: E402
from oracle import detector as OD  # noqa: E402


def _run_nms(pred, conf=0.01, iou=0.45, max_det=300, max_nms=30000, post=0, img=(640.0, 640.0), max_cand=None, geo=(1.0, 0.0, 0.0)):
    lib = sim()
    B, N, no = pred.shape
    max_cand = max_cand or N
    ws = np.zeros(lib.b2t_nms_workspace_bytes(B, max_cand, max_nms), dtype=np.uint8)
    out = np.zeros((B, max_det, 6), dtype=np.float32); cnt = np.zeros(B, dtype=np.int32)
    rc = lib.b2t_nms(ptr(pred), B, N, no, conf, iou, max_det, max_nms, max_cand, post, *geo, img[0], img[1], ptr(ws), ws.size, ptr(out),
                     ptr(cnt), None)
    assert rc == 0, lib.b2t_detect_last_error()
    return out, cnt


def _pred(seed, B, N, no, span=600.0, obj_shift=-1.0):
    g = torch.Generator().manual_seed(seed)
    p = torch.zeros((B, N, no))
    p[..., 0:2] = torch.rand((B, N, 2), generator=g) * span
    p[..., 2:4] = torch.rand((B, N, 2), generator=g) * 120 + 8
    p[..., 4] = torch.sigmoid(torch.randn((B, N), generator=g) * 1.5 + obj_shift)
    p[..., 5:] = torch.sigmoid(torch.randn((B, N, no - 5), generator=g))
    return p


def _check(out, cnt, ref, atol=1e-4):
    for b in range(len(ref)):
        n = int(cnt[b])
        assert n == ref[b].shape[0], (b, n, ref[b].shape[0])
        if n:
            assert np.array_equal(out[b, :n, 5], ref[b][:, 5].numpy())                      # same rows, same order
            assert np.allclose(out[b, :n, :5], ref[b][:, :5].numpy(), rtol=0, atol=atol)


def test_nms_pred_matches_reference_algorithm():
    B, N, no = 3, 1500, 11
    p = _pred(5, B, N, no)
    p[2, :, 4] = 0.0                                                 # an image without candidates -> (0, 6)
    out, cnt = _run_nms(np.ascontiguousarray(p.numpy()))
    ref = OD.non_max_suppression(p.clone(), conf_thres=0.01, iou_thres=0.45)
    assert int(cnt[0]) > 100 and int(cnt[2]) == 0
    _check(out, cnt, ref)


def test_nms_caps_max_det_and_post_processing():
    """dense scene: more than max_det survivors -> the greedy scan stops at the cap (general.py:680-681); post applies
    scale_coords / clip / round (track.py:239-240)."""
    B, N, no = 1, 2500, 8
    p = _pred(9, B, N, no, span=1200.0, obj_shift=1.0)
    p[..., 2:4] = p[..., 2:4] * 0.25
    out, cnt = _run_nms(np.ascontiguousarray(p.numpy()), max_det=50, post=1, img=(1000.0, 900.0))
    ref = OD.non_max_suppression(p.clone(), conf_thres=0.01, iou_thres=0.45, max_det=50)
    assert int(cnt[0]) == 50 == ref[0].shape[0]
    refp = [OD.post_process(ref[0], (900.0, 1000.0))]
    _check(out, cnt, refp)
    assert np.array_equal(out[0, :50, :4], np.round(out[0, :50, :4]))


def test_nms_ties_and_max_nms_truncation():
    """equal confidences (one histogram bin, exact in-bin ranking by row index) and n > max_nms."""
    B, N, no = 1, 700, 7
    p = _pred(3, B, N, no)
    p[0, :, 4] = 0.5
    p[0, :, 5:] = 0.0
    p[0, :, 5] = torch.tensor(np.repeat(np.linspace(0.9, 0.2, 7), 100).astype(np.float32))   # 7 groups of 100 ties
    out, cnt = _run_nms(np.ascontiguousarray(p.numpy()), max_nms=256)
    # reference semantics with a stable order: argsort(descending) on ties is unspecified in torch, so restate it stably
    x = p[0].clone()
    conf = (x[:, 5] * x[:, 4])
    order = np.lexsort((np.arange(N), -conf.numpy()))[:256]
    box = torch.stack([x[:, 0] - x[:, 2] / 2, x[:, 1] - x[:, 3] / 2, x[:, 0] + x[:, 2] / 2, x[:, 1] + x[:, 3] / 2], 1)[order]
    import torchvision
    keep = torchvision.ops.nms(box, conf[order], 0.45)     # ties: torchvision sorts by score too; kept set must match the stable order
    kept_rows = []
    boxes = box.numpy()
    for i in range(len(order)):                              # stable greedy restatement
        ok = True
        for j in kept_rows:
            a, c = boxes[j], boxes[i]
            iw = max(min(a[2], c[2]) - max(a[0], c[0]), 0.0); ih = max(min(a[3], c[3]) - max(a[1], c[1]), 0.0)
            inter = np.float32(iw) * np.float32(ih)
            u = np.float32((a[2] - a[0]) * (a[3] - a[1])) + np.float32((c[2] - c[0]) * (c[3] - c[1])) - inter
            if inter / u > 0.45:
                ok = False
                break
        if ok:
            kept_rows.append(i)
    kept_rows = kept_rows[:300]
    n = int(cnt[0])
    assert n == len(kept_rows)
    assert np.allclose(out[0, :n, :4], boxes[kept_rows], atol=1e-4)
    assert len(keep) >= 1


def test_detect_nms_fused_decode_matches_decode_then_nms():
    """b2t_detect_nms on raw head maps == Detect.forward decode (models/yolo.py:44-55) followed by NMS."""
    lib = sim()
    g = torch.Generator().manual_seed(21)
    B, no = 2, 9
    levels = [(8, 6, 8.0, [12, 16, 19, 36, 40, 28]), (4, 3, 16.0, [36, 75, 76, 55, 72, 146])]      # (h, w): non-square maps
    pitch = 32
    raws, preds, arr = [], [], (L.HeadLevel * len(levels))()
    off = 0
    for k, (h, w, stride, anc) in enumerate(levels):
        raw = torch.randn((B, h, w, pitch), generator=g)
        raw[..., 4::no] = raw[..., 4::no] * 1.5 - 0.5
        raws.append(np.ascontiguousarray(raw.numpy()))
        y = torch.sigmoid(raw[..., :3 * no].reshape(B, h, w, 3, no).permute(0, 3, 1, 2, 4))        # (B, 3, h, w, no)
        yv, xv = torch.meshgrid(torch.arange(h), torch.arange(w), indexing="ij")
        grid = torch.stack((xv, yv), 2).view(1, 1, h, w, 2).float()
        ag = torch.tensor(anc, dtype=torch.float32).view(1, 3, 1, 1, 2)
        y[..., 0:2] = (y[..., 0:2] * 2. - 0.5 + grid) * stride
        y[..., 2:4] = (y[..., 2:4] * 2) ** 2 * ag
        preds.append(y.reshape(B, -1, no))
        arr[k].raw = raws[k].ctypes.data; arr[k].raw_pitch = pitch; arr[k].h = h; arr[k].w = w; arr[k].stride = stride
        for j in range(6):
            arr[k].anchors[j] = float(anc[j])
        arr[k].level_off = off
        off += 3 * h * w
    pred = torch.cat(preds, 1)
    N = pred.shape[1]
    max_det, max_nms = 300, 30000
    ws = np.zeros(lib.b2t_nms_workspace_bytes(B, N, max_nms), dtype=np.uint8)
    out = np.zeros((B, max_det, 6), dtype=np.float32); cnt = np.zeros(B, dtype=np.int32)
    rc = lib.b2t_detect_nms(C.cast(arr, C.c_void_p), len(levels), B, no, 0.05, 0.45, max_det, max_nms, N, 0, 1.0, 0.0, 0.0, 64.0, 64.0,
                            ptr(ws), ws.size, ptr(out), ptr(cnt), None)
    assert rc == 0, lib.b2t_detect_last_error()
    ref = OD.non_max_suppression(pred.clone(), conf_thres=0.05, iou_thres=0.45)
    assert int(cnt[0]) > 10
    _check(out, cnt, ref, atol=2e-3)
    # and the same rows through the pred entry point
    out2, cnt2 = _run_nms(np.ascontiguousarray(pred.numpy()), conf=0.05)
    _check(out2, cnt2, ref)


def test_nms_argument_errors():
    lib = sim()
    p = np.zeros((1, 4, 8), dtype=np.float32)
    ws = np.zeros(lib.b2t_nms_workspace_bytes(1, 4, 4), dtype=np.uint8)
    out = np.zeros((1, 4, 6), dtype=np.float32); cnt = np.zeros(1, dtype=np.int32)
    assert lib.b2t_nms(ptr(p), 1, 4, 8, -0.5, 0.45, 4, 4, 4, 0, 1.0, 0.0, 0.0, 1.0, 1.0, ptr(ws), ws.size, ptr(out), ptr(cnt), None) != 0
    assert lib.b2t_nms(ptr(p), 1, 4, 8, 0.1, 0.45, 4, 4, 4, 0, 1.0, 0.0, 0.0, 1.0, 1.0, ptr(ws), 16, ptr(out), ptr(cnt), None) != 0
    assert b"workspace" in lib.b2t_detect_last_error()
    # fewer candidate slots than rows: refused (the surplus would be dropped in whatever order the atomics ran)
    assert lib.b2t_nms(ptr(p), 1, 4, 8, 0.1, 0.45, 4, 3, 3, 0, 1.0, 0.0, 0.0, 1.0, 1.0, ptr(ws), ws.size, ptr(out), ptr(cnt), None) == -1
    assert b"max_cand" in lib.b2t_detect_last_error()
    assert lib.b2t_nms(ptr(p), 1, 4, 8, 0.1, 0.45, 4, 4, 4, 1, 0.0, 0.0, 0.0, 1.0, 1.0, ptr(ws), ws.size, ptr(out), ptr(cnt), None) == -1


# ---------------------------------------------------------------- the edge cases of tests/nms_ref.py, bit for bit

def _check_bits(out, cnt, ref):
    for b, r in enumerate(ref):
        n = int(cnt[b])
        assert R.first_row_mismatch(out[b, :n], r["rows"]) is None, "image %d: first differing row %s (%d rows, expected %d)" % (
            b, R.first_row_mismatch(out[b, :n], r["rows"]), n, len(r["rows"]))


@pytest.mark.parametrize("name", sorted(R.edge_cases(large=False)))
def test_nms_edge_cases_bit_equal_nms_ref(name):
    pred, conf, iou, max_det, max_nms = R.edge_cases(large=False)[name]
    out, cnt = _run_nms(np.ascontiguousarray(pred), conf=conf, iou=iou, max_det=max_det, max_nms=max_nms)
    _check_bits(out, cnt, R.nms_ref(pred, conf, iou, max_det, max_nms))


@pytest.mark.parametrize("conf", [0.0, 0.25, 0.999])
@pytest.mark.parametrize("iou", [0.0, 0.45, 1.0])
@pytest.mark.parametrize("max_det", [1, 63, 64, 65, 300])
def test_nms_batch_of_edge_sizes_bit_equal_nms_ref(max_det, iou, conf):
    """B = 8 images of 0, 1, 63, 64, 65, 700, 64 and 1 candidates (block edges of the 64-row greedy scan)"""
    pred = R.batch_pred(sizes=(0, 1, 63, 64, 65, 700, 64, 1), N=900, nc=3)
    out, cnt = _run_nms(pred, conf=conf, iou=iou, max_det=max_det)
    _check_bits(out, cnt, R.nms_ref(pred, conf, iou, max_det, 30000))


@pytest.mark.parametrize("k", range(len(R.GEOMETRIES)))
def test_nms_post_geometry_in_band_and_reciprocal_form(k):
    """post = 1 with the scale_coords geometry of a letterboxed source: every coordinate inside the float64 band of
    tests/nms_ref.py, and equal to ``(x - pad) * (1 / gain)`` in fp32, clipped and rounded half to even"""
    src, canvas = R.GEOMETRIES[k]
    rows = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "scale_coords.npz"))["rows%d" % k]
    n = len(rows)
    pred = np.zeros((1, n, 6), np.float32)
    pred[0, :, 0] = (rows[:, 0] + rows[:, 2]) / 2; pred[0, :, 2] = rows[:, 2] - rows[:, 0]
    pred[0, :, 1] = (rows[:, 1] + rows[:, 3]) / 2; pred[0, :, 3] = rows[:, 3] - rows[:, 1]
    pred[0, :, 4] = np.linspace(0.99, 0.5, n, dtype=np.float32)
    pred[0, :, 5] = 1.0
    gain, pw, ph = R.scale_geometry(canvas, src)
    post0, cnt0 = _run_nms(pred, iou=1.0, max_det=300)
    post1, cnt1 = _run_nms(pred, iou=1.0, max_det=300, post=1, img=(float(src[1]), float(src[0])), geo=(gain, pw, ph))
    m = int(cnt0[0])
    assert m == int(cnt1[0]) == n
    got, base = post1[0, :m], post0[0, :m]
    lo, hi, _ = R.scale_coords_ref(base, canvas, src)
    assert len(R.outside_band(got, lo, hi)) == 0
    pad = np.array([pw, ph, pw, ph], np.float32)
    rec = np.round(np.clip(((base[:, :4] - pad) * (np.float32(1) / np.float32(gain))).astype(np.float32), 0,
                           np.array([src[1], src[0]] * 2, np.float32)))
    assert np.array_equal(got[:, :4], rec) and np.array_equal(got[:, 4:], base[:, 4:])
