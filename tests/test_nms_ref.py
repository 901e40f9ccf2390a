"""not-gpu: the float32 NMS reference and the float64 scale_coords reference (tests/nms_ref.py) agree with the reference's own
code -- torchvision's NMS through the oracle, and the reference's ``scale_coords`` through tests/golden/scale_coords.npz -- and the
comparisons built on them fail, at the right row, on each kind of bug the NMS stage or its post-processing could have."""
import os
import sys

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import nms_ref as R  # noqa: E402
from oracle import detector as OD  # noqa: E402

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "scale_coords.npz")


# ---------------------------------------------------------------- nms_ref == the reference's non_max_suppression (torchvision)

@pytest.mark.parametrize("seed,conf,iou,max_det,max_nms", [(0, 0.01, 0.45, 300, 30000), (1, 0.25, 0.45, 300, 30000), (2, 0.01, 0.6, 50, 30000),
                                                           (3, 0.01, 0.3, 300, 400), (4, 0.1, 0.45, 1, 30000)])
def test_nms_ref_equals_oracle_on_random_inputs(seed, conf, iou, max_det, max_nms):
    p = np.stack([R.random_pred(2500, seed * 10 + b, nc=6, span=700.0) for b in range(3)])
    p[2, :, 4] = 0.0                                                 # an image without candidates
    for b in range(2):                                               # no tied confidences: nudge the objectness of repeats up an ulp
        while True:
            rows, _, cf, _ = R.candidates(p[b], conf)
            _, first = np.unique(cf, return_index=True)
            dup = np.setdiff1d(np.arange(len(cf)), first)
            if not len(dup):
                break
            p[b, rows[dup], 4] = np.nextafter(p[b, rows[dup], 4], np.float32(2))
    ref = R.nms_ref(p, conf, iou, max_det, max_nms)
    for b, r in enumerate(ref):
        # the inputs must avoid the edges the oracle leaves open: ties in confidence, IoUs within rounding of the threshold
        rows, _, cf, _ = R.candidates(p[b], conf)
        assert len(np.unique(cf)) == len(cf), "tied confidences: torchvision's order is unspecified there"
        assert all(m > 1e-5 for _, _, _, m in r["decisions"]), "a pair within rounding of the threshold"
    orc = OD.non_max_suppression(torch.from_numpy(p.copy()), conf_thres=conf, iou_thres=iou, max_det=max_det, max_nms=max_nms)
    n_rows = 0
    for b in range(3):
        exp = orc[b].numpy()
        assert R.first_row_mismatch(ref[b]["rows"], exp) is None, "image %d" % b
        n_rows += len(exp)
        post = OD.post_process(orc[b], (700, 700)).numpy()                                     # same-size frames: gain 1, pad 0
        lo, hi, _ = R.scale_coords_ref(ref[b]["rows"], (700, 700), (700, 700))
        assert len(R.outside_band(post, lo, hi)) == 0 and np.array_equal(lo, hi)
    assert n_rows > (0 if max_det == 1 else 20)


def test_edge_cases_pin_what_they_claim():
    """the builders put rows where they say: IoU exactly at the fp32 threshold and one ulp either side, confidences at the
    threshold, the class offset joining boxes across 4096, and the max_nms cut through a run of ties"""
    for t in (0.45, 0.5, 0.7):
        pairs = R.iou_pair_boxes(t)
        assert sorted(pairs) == [-1, 0, 1]
        for k, (a, b) in pairs.items():
            assert R.iou32(a, b[None])[0] == {-1: np.nextafter(np.float32(t), np.float32(0)), 0: np.float32(t),
                                              1: np.nextafter(np.float32(t), np.float32(1))}[k]
        p, where = R.iou_pair_pred(t)
        r = R.nms_image(p, 0.01, t, 300, 30000)
        assert list(r["index"]) == [0, 1, 2, 3, 4]                   # only the pair one ulp above the threshold loses its second box
        bad = [d for d in r["decisions"] if d[1] != d[2]]
        assert all(m < R.IOU_BAND for _, _, _, m in bad)            # float64 may decide those pairs the other way, within rounding
    p = R.conf_edge_pred(0.25)
    rows, _, conf, _ = R.candidates(p, 0.25)
    assert (conf > np.float32(0.25)).all() and (p[:, 4] == np.float32(0.25)).any()
    assert list(R.nms_image(R.straddle_pred(), 0.01, 0.45, 300, 30000)["index"]) == [0, 2, 3]
    tp = R.tie_pred(3000, 1)
    r = R.nms_image(tp, 0.01, 0.45, 300, 1000)
    assert list(r["ranked"]) == list(range(1000)) and r["index"].max() < 1000


# ---------------------------------------------------------------- scale_coords: the golden of the reference's own function

def _golden():
    return np.load(GOLDEN)


@pytest.mark.parametrize("k", range(len(R.GEOMETRIES)))
def test_scale_coords_ref_and_dropin_match_reference_golden(k):
    from b200track.preprocess import scale_coords_geometry
    from utils.general import scale_coords
    g = _golden()
    src, canvas = tuple(int(v) for v in g["src"][k]), tuple(int(v) for v in g["canvas"][k])
    assert (src, canvas) == R.GEOMETRIES[k]
    assert scale_coords_geometry(canvas, src) == R.scale_geometry(canvas, src)
    rows = g["rows%d" % k]
    t = torch.from_numpy(rows.copy())
    t[:, :4] = scale_coords(canvas, t[:, :4], src).round()
    assert np.array_equal(t.numpy(), g["out%d" % k])                # the drop-in is the reference's function, bit for bit on the CPU
    lo, hi, v = R.scale_coords_ref(rows, canvas, src)
    for name in ("out%d", "out64_%d"):
        assert len(R.outside_band(g[name % k], lo, hi)) == 0, name % k
    out64 = g["out64_%d" % k][:, :4]
    decided = lo == hi
    assert np.array_equal(out64[decided], lo[decided])
    # the half-integer rows are what they claim: some coordinates sit within rounding of k + 0.5, some exactly on it
    n_half = len(R.half_integer_rows(canvas, src))
    assert (np.abs(v[:n_half] - np.floor(v[:n_half]) - 0.5) < 1e-3).sum() >= n_half


def test_scale_coords_cpu_float32_against_reciprocal_form():
    """torch divides a CPU float32 tensor by a Python scalar; on a CUDA tensor it multiplies by the fp32 reciprocal (the form the
    kernel follows).  At 1080p (gain 2/3) and 721 x 1283 (gain 0.997662) the engineered rows tell the two apart, inside the band."""
    g = _golden()
    differ = {}
    for k, (src, canvas) in enumerate(R.GEOMETRIES):
        rows = g["rows%d" % k]
        gain, pw, ph = R.scale_geometry(canvas, src)
        pad = np.array([pw, ph, pw, ph], np.float32)
        lim = np.array([src[1], src[0]] * 2, np.float32)
        rec = np.round(np.clip(((rows[:, :4] - pad) * (np.float32(1) / np.float32(gain))).astype(np.float32), 0, lim))
        lo, hi, _ = R.scale_coords_ref(rows, canvas, src)
        assert len(R.outside_band(rec, lo, hi)) == 0
        differ[(src, canvas)] = int((rec != g["out%d" % k][:, :4]).sum())
    print("\ncoordinates where CPU torch (division) and the reciprocal form round differently:", differ)
    assert differ[((1080, 1920), (768, 1280))] > 0                 # the rows reach the cases where the two forms part
    for k in (1, 2, 4, 5):                                           # powers-of-two gains: exact, no difference
        assert differ[R.GEOMETRIES[k]] == 0


# ---------------------------------------------------------------- the harness catches each bug, at the right row

def _ge(v, thr):
    return v >= np.float32(thr)


def _nms_variant(pred, conf, iou, max_det, max_nms, gt_filter=R.above, gt_iou=R.above, tie_desc=False, offset=True, cut_after=False):
    rows, box, cf, cls = R.candidates(pred, conf, gt=gt_filter)
    order = np.lexsort((-rows if tie_desc else rows, -cf.astype(np.float64)))
    if not cut_after:
        order = order[:max_nms]
    sbox = R.offset_boxes(box[order], cls[order]) if offset else box[order]
    kept, _ = R.greedy(sbox, iou, max_det, gt=gt_iou)
    if cut_after:
        kept = kept[:max_nms]
    sel = order[kept]
    return np.concatenate([box[sel], cf[sel, None], cls[sel, None]], 1).astype(np.float32)


def test_harness_catches_non_strict_filter():
    p = R.conf_edge_pred(0.25)
    exp = R.nms_image(p, 0.25, 0.45, 300, 30000)
    got = _nms_variant(p, 0.25, 0.45, 300, 30000, gt_filter=_ge)
    assert np.array_equal(_nms_variant(p, 0.25, 0.45, 300, 30000), exp["rows"])
    # the first row at exactly the threshold (obj = 0.25, class score 1: row 0) ranks after the rows above it
    first = int(np.sum(exp["rows"][:, 4] > np.float32(0.25)))
    assert R.first_row_mismatch(got, exp["rows"]) == first


def test_harness_catches_non_strict_iou():
    p, where = R.iou_pair_pred(0.45)
    exp = R.nms_image(p, 0.01, 0.45, 300, 30000)["rows"]
    got = _nms_variant(p, 0.01, 0.45, 300, 30000, gt_iou=_ge)
    assert R.first_row_mismatch(got, exp) == where[0][1]            # the second box of the pair exactly at the threshold


def test_harness_catches_ties_ranked_descending():
    p = R.tie_pred(3000, 1)
    exp = R.nms_image(p, 0.01, 0.45, 300, 1000)["rows"]
    got = _nms_variant(p, 0.01, 0.45, 300, 1000, tie_desc=True)
    assert R.first_row_mismatch(got, exp) == 0


@pytest.mark.parametrize("max_det", [1, 63, 64, 65])
def test_harness_catches_max_det_off_by_one(max_det):
    p = R.batch_pred(sizes=(5000,))[0]
    exp = R.nms_image(p, 0.01, 0.45, max_det, 30000)["rows"]
    assert len(exp) == max_det
    assert R.first_row_mismatch(_nms_variant(p, 0.01, 0.45, max_det + 1, 30000), exp) == max_det
    assert R.first_row_mismatch(_nms_variant(p, 0.01, 0.45, max_det - 1, 30000), exp) == max_det - 1


def test_harness_catches_max_nms_after_nms():
    def s():
        return [1.0]
    p = np.asarray([R._row(50, 50, 40, 40, 0.9, s()), R._row(52, 50, 40, 40, 0.8, s()), R._row(300, 300, 40, 40, 0.7, s())], np.float32)
    exp = R.nms_image(p, 0.01, 0.45, 300, 2)["rows"]                # rows 0, 1 ranked; 1 suppressed; row 2 cut before NMS
    assert len(exp) == 1
    assert R.first_row_mismatch(_nms_variant(p, 0.01, 0.45, 300, 2, cut_after=True), exp) == 1


def test_harness_catches_dropped_class_offset():
    p = R.straddle_pred()
    exp = R.nms_image(p, 0.01, 0.45, 300, 30000)["rows"]
    assert R.first_row_mismatch(_nms_variant(p, 0.01, 0.45, 300, 30000, offset=False), exp) == 2     # row 1 is no longer suppressed


def _flagged(got, lo, hi):
    bad = R.outside_band(got, lo, hi)
    return tuple(bad[0]) if len(bad) else None


def test_harness_catches_pad_subtracted_after_division():
    g = _golden()
    k = 0                                                            # 1080p: pad (0, 24)
    src, canvas = R.GEOMETRIES[k]
    rows = g["rows%d" % k]
    lo, hi, _ = R.scale_coords_ref(rows, canvas, src)
    blo, bhi, bv = R.scale_coords_ref(rows, canvas, src, pad_after_div=True)
    assert _flagged(np.round(bv), lo, hi) == (0, 1)                 # the first y coordinate: x has no pad


def test_harness_catches_clip_to_canvas():
    g = _golden()
    k = 0
    src, canvas = R.GEOMETRIES[k]
    rows = g["rows%d" % k]
    lo, hi, v = R.scale_coords_ref(rows, canvas, src)
    _, _, bv = R.scale_coords_ref(rows, canvas, src, clip_hw=canvas)
    over = v > np.array([canvas[1], canvas[0]] * 2) + 0.5             # past the canvas edge, inside the source frame
    assert over.any()
    assert _flagged(np.round(bv), lo, hi) == tuple(np.argwhere(over)[0])


def test_harness_catches_round_half_away_from_zero():
    g = _golden()
    k = 1                                                            # 720p: gain 1/2, exact ties at k + 0.5
    src, canvas = R.GEOMETRIES[k]
    rows = g["rows%d" % k]
    lo, hi, v = R.scale_coords_ref(rows, canvas, src)
    _, _, bv = R.scale_coords_ref(rows, canvas, src, half_away=True)
    bad = np.sign(bv) * np.floor(np.abs(bv) + 0.5)
    tie_even = (v - np.floor(v) == 0.5) & (np.floor(v) % 2 == 0)
    assert tie_even.any()
    assert _flagged(bad, lo, hi) == tuple(np.argwhere(tie_even)[0])
