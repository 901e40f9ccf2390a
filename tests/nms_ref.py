"""Plain NumPy restatement of the NMS stage (csrc/b2t_nms.cu) and of ``scale_coords(...).round()``, with the case builders that put
inputs exactly on the edges where that stage can go wrong.  TEST INFRASTRUCTURE; CPU only.

``nms_ref`` is the kernel's documented semantics, one operation at a time in float32:
  * filter: ``obj > thr``, the class scores times ``obj`` (one fp32 multiply each), the FIRST maximum, ``best > thr``
    (utils/general.py:616, :648, :658, :664; thresholds compared in fp32, as torch compares a float tensor with a Python scalar);
  * ``xywh2xyxy`` in fp32 (:265-272);
  * a STABLE total order: confidence descending, then row index ascending -- the kernel's tie rule (the reference's argsort and
    torchvision's order leave ties unspecified);
  * the first ``max_nms`` of that order, then class-offset boxes ``box + cls * max_wh`` in fp32 (:673-678);
  * greedy suppression with torchvision's ``devIoU``, each operation rounded on its own: ``inter / (sa + sb - inter) > thr``, up to
    ``max_det`` kept rows.
Every greedy decision is also made with the IoU in float64 from the same fp32 boxes; ``decisions`` lists them with the distance of
the closest IoU from the threshold, so a disagreement can be told apart from a decision that sits within rounding of it.

``scale_coords_ref`` is ``scale_coords(img1_shape, coords, img0_shape, ratio_pad=None)`` + clip + ``.round()`` (utils/general.py:319-340,
tracker/track.py:240) in float64: the integer each coordinate must round to, or both neighbours where the float64 value lies within
fp32 rounding of a half-integer."""
import numpy as np

F32 = np.float32
MAX_WH = 4096.0
IOU_BAND = 1e-6            # an fp32 IoU (five roundings of values <= the union) is within this of the float64 one


# ---------------------------------------------------------------- the NMS stage, piece by piece (tests recombine the pieces with one altered)

def above(v, thr):
    """the strict test of the filter and of the IoU (both are ``>``)"""
    return v > F32(thr)


def candidates(pred, conf_thres, gt=above):
    """pred (N, no) float32 -> (row index, xyxy boxes, conf, cls) of the rows that pass the filter, in row order"""
    pred = np.asarray(pred, F32)
    obj = pred[:, 4]
    ok = gt(obj, conf_thres)
    rows = np.nonzero(ok)[0]
    x = pred[rows]
    scores = x[:, 5:] * x[:, 4:5]                                   # fp32 products
    cls = np.argmax(scores, 1)                                       # the first maximum
    best = scores[np.arange(len(rows)), cls]
    keep = gt(best, conf_thres)
    rows, x, best, cls = rows[keep], x[keep], best[keep], cls[keep]
    half_w, half_h = x[:, 2] / F32(2), x[:, 3] / F32(2)
    box = np.stack([x[:, 0] - half_w, x[:, 1] - half_h, x[:, 0] + half_w, x[:, 1] + half_h], 1).astype(F32)
    return rows, box, best.astype(F32), cls.astype(F32)


def rank(conf, rows):
    """stable order: confidence descending, row index ascending"""
    return np.lexsort((rows, -conf.astype(np.float64)))


def offset_boxes(box, cls, max_wh=MAX_WH):
    return (box + (cls * F32(max_wh))[:, None]).astype(F32)


def iou32(a, b):
    """torchvision devIoU of box a against boxes b, fp32, every operation rounded on its own"""
    left, right = np.maximum(a[0], b[:, 0]), np.minimum(a[2], b[:, 2])
    top, bottom = np.maximum(a[1], b[:, 1]), np.minimum(a[3], b[:, 3])
    w = np.maximum(F32(right - left), F32(0)); h = np.maximum(F32(bottom - top), F32(0))
    inter = F32(w * h)
    sa = F32(F32(a[2] - a[0]) * F32(a[3] - a[1]))
    sb = F32(F32(b[:, 2] - b[:, 0]) * F32(b[:, 3] - b[:, 1]))
    with np.errstate(invalid="ignore", divide="ignore"):
        return F32(inter / F32(F32(sa + sb) - inter))


def iou64(a, b):
    a, b = a.astype(np.float64), b.astype(np.float64)
    w = np.maximum(np.minimum(a[2], b[:, 2]) - np.maximum(a[0], b[:, 0]), 0.0)
    h = np.maximum(np.minimum(a[3], b[:, 3]) - np.maximum(a[1], b[:, 1]), 0.0)
    inter = w * h
    with np.errstate(invalid="ignore", divide="ignore"):
        return inter / ((a[2] - a[0]) * (a[3] - a[1]) + (b[:, 2] - b[:, 0]) * (b[:, 3] - b[:, 1]) - inter)


def greedy(sbox, iou_thres, max_det, gt=above):
    """kept positions of the ranked class-offset boxes, and one decision record per visited position:
    (position, kept, kept with float64 IoUs against the same kept set, min |IoU64 - thr| over the kept boxes)"""
    kept, decisions = [], []
    thr64 = float(F32(iou_thres))
    for i in range(len(sbox)):
        if len(kept) >= max_det:
            break
        if kept:
            kb = sbox[kept]
            i32, i64 = iou32(sbox[i], kb), iou64(sbox[i], kb)
            keep = not bool(gt(i32, iou_thres).any())
            keep64 = not bool((i64 > thr64).any())
            with np.errstate(invalid="ignore"):
                margin = float(np.nanmin(np.abs(i64 - thr64))) if np.isfinite(i64).any() else np.inf
        else:
            keep = keep64 = True
            margin = np.inf
        decisions.append((i, keep, keep64, margin))
        if keep:
            kept.append(i)
    return np.asarray(kept, np.int64), decisions


def nms_image(pred, conf_thres, iou_thres, max_det, max_nms, max_wh=MAX_WH):
    """one image: dict(rows = (n, 6) float32 [x1 y1 x2 y2 conf cls], index = source row of each, decisions, ranked = the candidates
    after the max_nms cut, in rank order)"""
    rows, box, conf, cls = candidates(pred, conf_thres)
    order = rank(conf, rows)[:max_nms]
    sbox = offset_boxes(box[order], cls[order], max_wh)
    kept, decisions = greedy(sbox, iou_thres, max_det)
    sel = order[kept]
    out = np.concatenate([box[sel], conf[sel, None], cls[sel, None]], 1).astype(F32) if len(sel) else np.zeros((0, 6), F32)
    return dict(rows=out, index=rows[sel], decisions=decisions, ranked=rows[order])


def nms_ref(pred, conf_thres, iou_thres, max_det, max_nms, max_wh=MAX_WH):
    """pred (B, N, no) float32 -> per image the dict of ``nms_image``"""
    return [nms_image(p, conf_thres, iou_thres, max_det, max_nms, max_wh) for p in np.asarray(pred, F32)]


def first_row_mismatch(got, exp):
    """got / exp: (n, 6) float32 rows.  The first row index at which they differ bit for bit (a shorter list differs at its
    length), or None."""
    n = min(len(got), len(exp))
    g, e = np.ascontiguousarray(got[:n], F32).view(np.int32), np.ascontiguousarray(exp[:n], F32).view(np.int32)
    bad = np.nonzero((g != e).any(1))[0]
    if len(bad):
        return int(bad[0])
    return None if len(got) == len(exp) else n


# ---------------------------------------------------------------- scale_coords + clip + round in float64

def scale_geometry(canvas_hw, src_hw):
    """gain and pad exactly as utils/general.py:322-323 computes them (Python floats)"""
    gain = min(canvas_hw[0] / src_hw[0], canvas_hw[1] / src_hw[1])
    return gain, (canvas_hw[1] - src_hw[1] * gain) / 2, (canvas_hw[0] - src_hw[0] * gain) / 2


def scale_coords_ref(rows, canvas_hw, src_hw, pad_after_div=False, clip_hw=None, half_away=False):
    """rows (n, >= 4) float32 canvas boxes -> (lo, hi, value) float64 (n, 4): every coordinate must round to an integer in
    [lo, hi]; lo == hi except where the float64 value lies within fp32 rounding (3 ulps of the operands' scale) of a half-integer.
    pad_after_div / clip_hw / half_away: deliberate bugs for the harness tests (pad subtracted after the division, clipping to
    another size, rounding half away from zero)."""
    gain, padw, padh = scale_geometry(canvas_hw, src_hw)
    x = np.asarray(rows, F32)[:, :4].astype(np.float64)
    pad = np.array([padw, padh, padw, padh])
    v = x / gain - pad if pad_after_div else (x - pad) / gain
    ch, cw = src_hw if clip_hw is None else clip_hw
    v = np.clip(v, 0.0, np.array([cw, ch, cw, ch], np.float64))
    if half_away:
        r = np.sign(v) * np.floor(np.abs(v) + 0.5)
    else:
        r = np.round(v)                                              # half to even, like torch.round
    # fp32 evaluation error: pad -> fp32, x - pad, the division (or reciprocal and multiply) -- at most 3 ulps of the larger of
    # |v| and |pad| / gain.  None at all when gain is a power of two, pad an fp32 value and x - pad exact in fp32: those
    # coordinates (also exact ties k + 0.5) have one answer
    d = x - pad
    exact = (np.frexp(gain)[0] == 0.5) & (F32(pad) == pad) & (d.astype(F32) == d)
    scale = np.maximum(np.abs(v), np.abs(pad) / gain).astype(F32)
    tol = np.where(exact, 0.0, 3.0 * np.spacing(scale).astype(np.float64))
    frac = v - np.floor(v)
    near = (tol > 0) & (np.abs(frac - 0.5) <= tol)
    lo = np.where(near, np.floor(v), r)
    hi = np.where(near, np.floor(v) + 1.0, r)
    return lo, hi, v


def outside_band(got, lo, hi):
    """(row, column) pairs of got (n, >= 4) that lie outside [lo, hi]"""
    g = np.asarray(got, np.float64)[:, :4]
    return np.argwhere((g < lo) | (g > hi))


# ---------------------------------------------------------------- case builders: pred rows (cx cy w h obj cls...) fixed exactly

def _row(cx, cy, w, h, obj, cls_scores):
    return [F32(cx), F32(cy), F32(w), F32(h), F32(obj)] + [F32(c) for c in cls_scores]


def exact_xywh(x1, x2):
    """(cx, w) float32 with cx - w/2 == x1 and cx + w/2 == x2 in fp32, or None"""
    x1, x2 = F32(x1), F32(x2)
    w = F32(x2 - x1)
    cx = F32((np.float64(x1) + np.float64(x2)) / 2)
    if F32(cx - w / F32(2)) == x1 and F32(cx + w / F32(2)) == x2:
        return cx, w
    return None


def conf_edge_pred(conf_thres, nc=3, n_grid=6):
    """rows at conf_thres and one ulp either side, through obj alone (cls score 1) and through the product obj * cls; boxes on a
    grid that never overlap.  Returns (N, 5 + nc) float32."""
    t = F32(conf_thres)
    dn, up = np.nextafter(t, F32(-1)), np.nextafter(t, F32(2))
    objs = [t, dn, up]
    rows, k = [], 0
    for o in objs:                                                   # obj at the edge, class score exactly 1
        for c in range(nc):
            s = [F32(0.0)] * nc
            s[c] = F32(1.0)
            rows.append(_row(40 + 100 * (k % n_grid), 40 + 100 * (k // n_grid), 30, 30, o, s)); k += 1
    for o in objs:                                                   # obj = 1, best class score at the edge (product = the score)
        s = [F32(0.0)] * nc
        s[k % nc] = o
        rows.append(_row(40 + 100 * (k % n_grid), 40 + 100 * (k // n_grid), 30, 30, F32(1.0), s)); k += 1
    # obj above the edge, product lands on it or beside it after fp32 rounding; two classes tied at the maximum (first wins)
    for o in (np.nextafter(t, F32(2)), F32(min(1.0, float(t) * 2 + 0.01))):
        for sc in (F32(t / o), np.nextafter(F32(t / o), F32(2)), np.nextafter(F32(t / o), F32(-1))):
            s = [sc] * nc
            rows.append(_row(40 + 100 * (k % n_grid), 40 + 100 * (k // n_grid), 30, 30, o, s)); k += 1
    return np.asarray(rows, F32)


def iou_pair_boxes(iou_thres, width=58.0, height=40.0, span=48):
    """{-1, 0, +1: (a, b)}: two float32 xyxy boxes (class 0) whose fp32 IoU is the fp32 threshold, one ulp below it, one above it --
    found by stepping b's corners an ulp at a time around the exact solution of (W - d) / (W + d) = thr."""
    t = F32(iou_thres)
    want = {-1: np.nextafter(t, F32(-1)), 0: t, 1: np.nextafter(t, F32(2))}
    d0 = width * (1 - float(t)) / (1 + float(t))
    a = np.array([0, 0, width, height], F32)
    found = {}
    x1 = F32(d0)
    for s1 in range(-span, span + 1):
        bx1 = x1
        for _ in range(abs(s1)):
            bx1 = np.nextafter(bx1, F32(np.sign(s1) * 1e9))
        bx2 = F32(np.float64(bx1) + width)
        for s2 in range(-4, 5):
            cx2 = bx2
            for _ in range(abs(s2)):
                cx2 = np.nextafter(cx2, F32(np.sign(s2) * 1e9))
            if exact_xywh(bx1, cx2) is None:
                continue
            b = np.array([bx1, 0, cx2, height], F32)
            v = iou32(a, b[None])[0]
            for k, w in want.items():
                if k not in found and v == w:
                    found[k] = (a, b)
        if len(found) == 3:
            break
    return found


def iou_pair_pred(iou_thres, nc=2):
    """pred rows of the three threshold pairs (stacked 100 px apart in y, the first box of each pair more confident).  Returns
    (pred (6, 5 + nc) float32, {-1/0/+1: (row of the first box, row of the second)})."""
    pairs = iou_pair_boxes(iou_thres)
    rows, where = [], {}
    for n, (k, (a, b)) in enumerate(sorted(pairs.items())):
        y = F32(100 * n)
        for j, (box, conf) in enumerate(((a, 0.9 - 0.1 * n), (b, 0.85 - 0.1 * n))):
            cx, w = exact_xywh(box[0], box[2])
            s = [F32(0.0)] * nc
            s[0] = F32(1.0)
            rows.append(_row(cx, y + box[3] / 2, w, box[3], conf, s))
        where[k] = (2 * n, 2 * n + 1)
    return np.asarray(rows, F32), where


def straddle_pred(nc=3):
    """boxes past 4096 px: a class-0 box at (4090, 4126)-(4110, 4166) and a class-1 box at (-6, 30)-(14, 70) coincide once the class
    offset (cls * 4096, added to all four coordinates) is in -- the reference's class-offset NMS suppresses across the two classes there -- plus a class-0 box
    across x = 4096 and a class-1 box that does not reach it."""
    def cls(c):
        s = [F32(0.0)] * nc
        s[c] = F32(0.9)
        return s
    rows = [_row(4100, 4146, 20, 40, 1.0, cls(0)),      # [4090, 4126, 4110, 4166]
            _row(4, 50, 20, 40, 0.95, cls(1)),          # [-6, 30, 14, 70] + 4096: the same box after the offset
            _row(4096, 200, 30, 30, 1.0, cls(0)),       # across 4096
            _row(100, 200, 30, 30, 0.5, cls(1))]        # no partner
    return np.asarray(rows, F32)


def tie_pred(n, seed=0, nc=1, span=1200.0, conf=1.0):
    """n rows at confidence exactly ``conf`` (obj = conf, class score 1), random boxes"""
    rng = np.random.default_rng(seed)
    p = np.zeros((n, 5 + nc), F32)
    p[:, 0:2] = rng.uniform(0, span, (n, 2))
    p[:, 2:4] = rng.uniform(4, 60, (n, 2))
    p[:, 4] = conf
    p[:, 5] = 1.0
    return p


def random_pred(n, seed, nc=5, span=640.0, obj_shift=-1.0, wh=(8, 128)):
    rng = np.random.default_rng(seed)
    p = np.zeros((n, 5 + nc), F32)
    p[:, 0:2] = rng.uniform(0, span, (n, 2))
    p[:, 2:4] = rng.uniform(wh[0], wh[1], (n, 2))
    p[:, 4] = 1 / (1 + np.exp(-(rng.standard_normal(n) * 1.5 + obj_shift)))
    p[:, 5:] = 1 / (1 + np.exp(-rng.standard_normal((n, nc))))
    return p


def zero_area_pred(nc=2):
    """zero-width, zero-height and point boxes (0 / 0 IoU is NaN: never above the threshold) next to ordinary ones"""
    def s():
        return [F32(1.0)] + [F32(0.0)] * (nc - 1)
    return np.asarray([_row(50, 50, 0, 20, 0.9, s()), _row(50, 50, 0, 20, 0.8, s()),       # same zero-width box twice
                       _row(80, 80, 10, 0, 0.7, s()), _row(80, 80, 0, 0, 0.6, s()),
                       _row(50, 50, 20, 20, 0.5, s()), _row(80, 80, 20, 20, 0.4, s())], F32)


def half_integer_rows(canvas_hw, src_hw, ks=(0, 1, 2, 3, 10, 11, 100, 101, 500, 501), steps=(0, 1, 2, 4, 8, 16)):
    """canvas boxes whose scaled coordinates land on k + 0.5 (the nearest float32) and ``steps`` ulps either side, for every
    coordinate; clipped values (k + 0.5 beyond the source size) are skipped.  Returns (n, 6) float32 rows (conf 0.5, cls 0)."""
    gain, padw, padh = scale_geometry(canvas_hw, src_hw)
    h, w = src_hw
    xs = []
    for pad, lim in ((padw, w), (padh, h)):
        vals = []
        for k in ks:
            if k + 0.5 > lim:
                continue
            c = F32((k + 0.5) * gain + pad)
            for s in sorted(set(steps) | {-t for t in steps}):
                v = c
                for _ in range(abs(s)):
                    v = np.nextafter(v, F32(np.sign(s) * 1e9))
                vals.append(v)
        xs.append(np.asarray(vals, F32))
    n = max(len(xs[0]), len(xs[1]))
    xv, yv = np.resize(xs[0], n), np.resize(xs[1], n)
    rows = np.zeros((n, 6), F32)
    rows[:, 0], rows[:, 1] = np.minimum(xv, xv[::-1]), np.minimum(yv, yv[::-1])
    rows[:, 2], rows[:, 3] = np.maximum(xv, xv[::-1]), np.maximum(yv, yv[::-1])
    rows[:, 4] = 0.5
    return rows


# the geometries of tests/golden/scale_coords.npz: (source (h, w), canvas (h, w))
GEOMETRIES = [((1080, 1920), (768, 1280)), ((720, 1280), (384, 640)), ((360, 640), (384, 640)), ((721, 1283), (768, 1280)),
              ((480, 640), (960, 1280)), ((640, 640), (640, 640))]


def batch_pred(sizes=(0, 1, 63, 64, 65, 5000, 64, 1), N=6000, nc=5, seed=0):
    """B = len(sizes) images of N rows; image b has sizes[b] rows that pass any conf_thres < 0.5 (obj 0.9, class scores >= 0.6:
    the rest have obj 0), boxes dense enough that the greedy scan suppresses; the large image also carries rows with
    confidence above 1 and rows at exactly 1.0"""
    rng = np.random.default_rng(seed)
    p = np.zeros((len(sizes), N, 5 + nc), F32)
    for b, n in enumerate(sizes):
        p[b] = random_pred(N, seed + b, nc=nc, span=400.0 if n > 100 else 640.0, wh=(8, 96))
        p[b, :, 4] = 0.0
        sel = rng.permutation(N)[:n]
        p[b, sel, 4] = rng.uniform(0.9, 0.9999, n)
        p[b, sel, 5:] = rng.uniform(0.6, 1.0, (n, nc))
        if n > 1000:
            p[b, sel[:40], 4] = rng.uniform(1.0, 1.5, 40)            # conf > 1 (pred rows are not clamped)
            p[b, sel[40:80], 4] = 1.0
            p[b, sel[40:80], 5:] = 0.0
            p[b, sel[40:80], 5] = 1.0                                 # conf exactly 1.0, ties
    return p


def edge_cases(large=True):
    """name -> (pred (B, N, no) float32, conf_thres, iou_thres, max_det, max_nms).  large=False leaves out the 102 000-row tie
    image (its in-bin ranking is quadratic: too slow for the host simulator) and shrinks the batch."""
    c = {}
    for t in (0.45, 0.5, 0.7):
        p, _ = iou_pair_pred(t)
        c["iou_pairs_%g" % t] = (p[None], 0.01, t, 300, 30000)
    for t in (0.0, 0.01, 0.25, 0.999):
        p = conf_edge_pred(t)                                         # t = 0: obj of +-1 denormal ulp and exactly 0
        c["conf_edges_%g" % t] = (p[None], t, 0.45, 300, 30000)
    c["straddle_4096"] = (straddle_pred()[None], 0.01, 0.45, 300, 30000)
    c["zero_area"] = (zero_area_pred()[None], 0.01, 0.45, 300, 30000)
    c["zero_area_iou0"] = (zero_area_pred()[None], 0.01, 0.0, 300, 30000)
    p = tie_pred(3000, 1)
    c["ties_3000_max_nms_1000"] = (p[None], 0.01, 0.45, 300, 1000)
    c["ties_conf_above_one"] = (tie_pred(500, 2, conf=1.25)[None], 0.01, 0.45, 64, 30000)
    if large:
        c["ties_102000_max_nms_30000"] = (tie_pred(102000, 3, span=4000.0)[None], 0.01, 0.45, 300, 30000)
        c["ties_102000_max_det_2048"] = (tie_pred(102000, 4, span=4000.0)[None], 0.01, 0.45, 2048, 30000)
    return c
