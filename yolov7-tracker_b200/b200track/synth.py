"""Seeded synthetic detection streams (SURVEY.md section 8d "Synthetic inputs").

There is no dataset and no detector checkpoint in the reference (weights/ has no YOLO
weights), so every tracker-side test, golden fixture and bench line is driven by these
streams.  A stream is what ``tracker/track.py:149`` hands to ``tracker.update``: per frame an
``(n, 6)`` float32 array ``[x1, y1, x2, y2, score, cls]`` with integer-rounded, clipped
coordinates (q9) sorted by descending score (q13: NMS output order).
"""
import hashlib

import numpy as np


def make_stream(seed, n_frames, n_obj=300, img=1280, miss=0.05, warp_sigma=0.0):
    """Returns (frames, warps): list of (n_i, 6) float32 arrays and a (n_frames, 2, 3) float64
    array of per-frame camera warps (identity rotation, N(0, warp_sigma) translation)."""
    rng = np.random.default_rng(seed)
    cx = rng.uniform(200, img - 200, n_obj)
    cy = rng.uniform(200, img - 200, n_obj)
    w = rng.uniform(20, 80, n_obj)
    h = rng.uniform(40, 160, n_obj)
    vx = rng.normal(0, 1, n_obj)
    vy = rng.normal(0, 1, n_obj)
    cls = rng.integers(0, 3, n_obj).astype(np.float32)
    frames = []
    warps = np.zeros((n_frames, 2, 3), dtype=np.float64)
    warps[:, 0, 0] = warps[:, 1, 1] = 1.0
    cam = np.zeros(2)
    for f in range(n_frames):
        cx += vx
        cy += vy
        # bounce on the borders so the population stays inside the frame
        bx = (cx < 60) | (cx > img - 60)
        by = (cy < 60) | (cy > img - 60)
        vx[bx] = -vx[bx]
        vy[by] = -vy[by]
        if warp_sigma > 0:
            t = rng.normal(0, warp_sigma, 2)
            warps[f, :, 2] = t
            cam += t
        jit = rng.normal(0, 1, (n_obj, 4))
        score = rng.uniform(0.05, 0.95, n_obj).astype(np.float32)
        keep = rng.uniform(0, 1, n_obj) >= miss
        x1 = cx - w / 2 + jit[:, 0] + cam[0]
        y1 = cy - h / 2 + jit[:, 1] + cam[1]
        x2 = cx + w / 2 + jit[:, 2] + cam[0]
        y2 = cy + h / 2 + jit[:, 3] + cam[1]
        box = np.stack([x1, y1, x2, y2], 1)
        box = np.round(np.clip(box, 0, img))
        ok = keep & ((box[:, 2] - box[:, 0]) >= 4) & ((box[:, 3] - box[:, 1]) >= 4)
        d = np.concatenate([box[ok], score[ok, None], cls[ok, None]], 1).astype(np.float32)
        order = np.argsort(-d[:, 4], kind="stable")
        frames.append(np.ascontiguousarray(d[order]))
    return frames, warps


def make_reid_stream(seed, n_frames, n_obj=60, feat_dim=64, img=1280, warp_sigma=1.0, occl=0.04):
    """A stream for BoT-SORT with appearance features: (frames, feats, warps).  feats[f] is an (n_i, feat_dim) float32 array aligned
    with the rows of frames[f] (the tracker reads only those of the high-score rows).
      * half of the objects move in pairs that cross each other head-on at the same height, so IoU alone can swap them;
      * every object has a seeded identity vector; a detection's feature is that vector plus noise, times a random scale in
        [0.3, 3] -- the extractor's features are not assumed to be unit vectors;
      * an object goes unseen for 3-8 frames with probability `occl` per frame (Lost tracks that are re-activated later);
      * about 15 % of the detections score in [0.1, 0.2) (low-score association, no feature).
    Coordinates are not rounded, so no two costs tie exactly."""
    rng = np.random.default_rng(seed)
    n_pair = n_obj // 4
    cx = rng.uniform(150, img - 150, n_obj)
    cy = rng.uniform(150, img - 150, n_obj)
    w = rng.uniform(30, 70, n_obj)
    h = rng.uniform(60, 140, n_obj)
    vx = rng.normal(0, 1.5, n_obj)
    vy = rng.normal(0, 1.5, n_obj)
    for k in range(n_pair):                                   # objects 2k and 2k+1 cross half-way through the stream
        a, b = 2 * k, 2 * k + 1
        speed = rng.uniform(2.0, 5.0)
        mid = rng.uniform(300, img - 300)
        cx[a], cx[b] = mid - speed * n_frames / 2, mid + speed * n_frames / 2
        cy[b] = cy[a] + rng.normal(0, 3)
        vx[a], vx[b], vy[a], vy[b] = speed, -speed, 0.0, 0.0
        w[b], h[b] = w[a] * rng.uniform(0.9, 1.1), h[a] * rng.uniform(0.9, 1.1)
    ident = rng.normal(0, 1, (n_obj, feat_dim))
    base_score = rng.uniform(0.35, 0.95, n_obj)
    hidden = np.zeros(n_obj, np.int64)
    frames, feats = [], []
    warps = np.zeros((n_frames, 2, 3), dtype=np.float64)
    warps[:, 0, 0] = warps[:, 1, 1] = 1.0
    cam = np.zeros(2)
    for f in range(n_frames):
        cx += vx
        cy += vy
        t = rng.normal(0, warp_sigma, 2)
        warps[f, :, 2] = t
        cam += t
        start = (hidden == 0) & (rng.uniform(0, 1, n_obj) < occl)
        hidden[start] = rng.integers(3, 9, int(start.sum()))
        seen = hidden == 0
        hidden[~seen] -= 1
        jit = rng.normal(0, 1.0, (n_obj, 4))
        score = np.where(rng.uniform(0, 1, n_obj) < 0.15, rng.uniform(0.1, 0.2, n_obj), base_score + rng.normal(0, 0.02, n_obj))
        x1 = cx - w / 2 + jit[:, 0] + cam[0]
        y1 = cy - h / 2 + jit[:, 1] + cam[1]
        x2 = cx + w / 2 + jit[:, 2] + cam[0]
        y2 = cy + h / 2 + jit[:, 3] + cam[1]
        box = np.clip(np.stack([x1, y1, x2, y2], 1), 0, img)
        ok = seen & ((box[:, 2] - box[:, 0]) >= 4) & ((box[:, 3] - box[:, 1]) >= 4)
        d = np.concatenate([box[ok], score[ok, None], (np.arange(n_obj) % 3)[ok, None]], 1).astype(np.float32)
        fe = (ident[ok] + rng.normal(0, 0.6, (int(ok.sum()), feat_dim))) * rng.uniform(0.3, 3.0, (int(ok.sum()), 1))
        fe = fe.astype(np.float32)
        order = np.argsort(-d[:, 4], kind="stable")
        frames.append(np.ascontiguousarray(d[order]))
        feats.append(np.ascontiguousarray(fe[order]))
    return frames, feats, warps


def make_strongsort_stream(seed, n_frames, n_obj=40, feat_dim=64, img=1280, warp_sigma=1.0, occl=0.04, jump=0.03):
    """A stream for StrongSORT: (frames, feats, warps), feats[f] row-aligned with frames[f].
      * every object has a seeded unit identity vector; a detection's feature is that vector plus noise, times a scale in [0.85, 1.15],
        so the raw features have norms around 1 and the Euclidean appearance term decides matches (StrongSORT compares raw detection
        rows with unit track rows, q19);
      * an object jumps by 1.5-3 box widths with probability `jump` per frame (0.4 on the frame after it enters), so that only
        appearance can match it (zero IoU), and
        goes unseen for 2-8 frames with probability `occl` (Lost tracks, re-activated wherever they reappear);
      * objects enter at staggered frames, so that unconfirmed tracks meet association 3 throughout the stream;
      * scores lie in [0.05, 0.95]: some rows fall below det_thresh (StrongSORT drops them) and some between det_thresh and
        det_thresh + 0.1 (no birth).
    Coordinates are not rounded, so no two costs tie exactly."""
    rng = np.random.default_rng(seed)
    cx = rng.uniform(150, img - 150, n_obj)
    cy = rng.uniform(150, img - 150, n_obj)
    w = rng.uniform(30, 70, n_obj)
    h = rng.uniform(60, 140, n_obj)
    vx = rng.normal(0, 2.0, n_obj)
    vy = rng.normal(0, 2.0, n_obj)
    ident = rng.normal(0, 1, (n_obj, feat_dim))
    ident /= np.linalg.norm(ident, axis=1, keepdims=True)
    enter = rng.integers(0, max(1, n_frames // 2), n_obj)
    enter[: n_obj // 3] = 0
    base_score = rng.uniform(0.3, 0.95, n_obj)
    hidden = np.zeros(n_obj, np.int64)
    frames, feats = [], []
    warps = np.zeros((n_frames, 2, 3), dtype=np.float64)
    warps[:, 0, 0] = warps[:, 1, 1] = 1.0
    cam = np.zeros(2)
    for f in range(n_frames):
        jmp = rng.uniform(0, 1, n_obj) < np.where(f == enter + 1, 0.4, jump)     # often right after a birth (association 3)
        ang = rng.uniform(0, 2 * np.pi, n_obj)
        dist = rng.uniform(1.5, 3.0, n_obj) * w
        cx += vx + jmp * dist * np.cos(ang)
        cy += vy + jmp * dist * np.sin(ang)
        cx = np.clip(cx, 80, img - 80)
        cy = np.clip(cy, 80, img - 80)
        t = rng.normal(0, warp_sigma, 2)
        warps[f, :, 2] = t
        cam += t
        start = (hidden == 0) & (rng.uniform(0, 1, n_obj) < occl)
        hidden[start] = rng.integers(2, 9, int(start.sum()))
        seen = (hidden == 0) & (enter <= f)
        hidden[hidden > 0] -= 1
        jit = rng.normal(0, 1.0, (n_obj, 4))
        score = np.clip(base_score + rng.normal(0, 0.05, n_obj), 0.05, 0.95)
        score = np.where(rng.uniform(0, 1, n_obj) < 0.1, rng.uniform(0.05, 0.2, n_obj), score)
        x1 = cx - w / 2 + jit[:, 0] + cam[0]
        y1 = cy - h / 2 + jit[:, 1] + cam[1]
        x2 = cx + w / 2 + jit[:, 2] + cam[0]
        y2 = cy + h / 2 + jit[:, 3] + cam[1]
        box = np.clip(np.stack([x1, y1, x2, y2], 1), 0, img)
        ok = seen & ((box[:, 2] - box[:, 0]) >= 4) & ((box[:, 3] - box[:, 1]) >= 4)
        d = np.concatenate([box[ok], score[ok, None], (np.arange(n_obj) % 3)[ok, None]], 1).astype(np.float32)
        k = int(ok.sum())
        fe = (ident[ok] + rng.normal(0, 0.25 / np.sqrt(feat_dim), (k, feat_dim))) * rng.uniform(0.85, 1.15, (k, 1))
        order = rng.permutation(k)
        frames.append(np.ascontiguousarray(d[order]))
        feats.append(np.ascontiguousarray(fe.astype(np.float32)[order]))
    return frames, feats, warps


def lifecycle_stream(seed, n_frames, n_obj=40, img=1280, conf_thresh=0.2, warp_sigma=0.0):
    """A stream that walks the tracker through its whole track life cycle: (frames, warps) like ``make_stream``.
      * a third of the objects are there from frame 1, the others are born at staggered frames; about half leave before the end;
      * every visible object starts an occlusion with p = 0.03 per frame, 2-45 frames long: the long ones outlive any
        ``max_time_lost`` up to 30 frames (the track is pruned), the shorter ones are re-found after a gap;
      * a quarter of the objects are twins of an earlier one (offset by 1-2 px, same size and motion): when one twin is occluded its
        Lost track sits on top of the other's Tracked one, so ``remove_duplicate_stracks`` drops one of them.  A twin's top-left
        corner lies a quarter pixel off the integer grid, so its box never has the same area as its sibling's and no track box
        is exactly as close to both (an exact cost tie would make the assignment solver-dependent);
      * four frames (never the first) carry no detection at all;
      * about 5 % of the scores are exactly ``float32(conf)``, ``float32(max(0.15, conf - 0.3))`` or ``float32(conf + 0.1)`` -- the
        high / low / new-track thresholds the trackers compare against;
      * warp_sigma > 0: per-frame camera warps with a small rotation and scale and N(0, warp_sigma) translation (boxes move with the
        translation).
    Coordinates are integer-rounded (twins' top-left corners: plus a quarter pixel) and clipped, and every frame is sorted by
    descending score, like ``make_stream``."""
    rng = np.random.default_rng(seed)
    n_twin = n_obj // 4
    n_base = n_obj - n_twin
    cx = rng.uniform(150, img - 150, n_obj)
    cy = rng.uniform(150, img - 150, n_obj)
    w = rng.uniform(24, 80, n_obj)
    h = rng.uniform(48, 160, n_obj)
    vx = rng.normal(0, 1, n_obj)
    vy = rng.normal(0, 1, n_obj)
    cls = rng.integers(0, 3, n_obj).astype(np.float32)
    base_score = rng.uniform(0.25, 0.95, n_obj)
    born = np.where(rng.uniform(0, 1, n_obj) < 1 / 3, 0, rng.integers(1, max(2, int(0.7 * n_frames)), n_obj))
    life = rng.integers(max(2, n_frames // 4), 2 * n_frames, n_obj)
    twin_of = rng.choice(n_base, n_twin, replace=False)
    for k, a in enumerate(twin_of):                            # a twin copies an earlier object's box and motion
        b = n_base + k
        cx[b], cy[b] = cx[a] + rng.integers(1, 3), cy[a] + rng.integers(1, 3)
        w[b], h[b], vx[b], vy[b], cls[b] = w[a], h[a], vx[a], vy[a], cls[a]
        born[b] = born[a] + rng.integers(0, 8)
    died = born + life
    empty = set((1 + rng.choice(n_frames - 1, min(4, n_frames - 1), replace=False)).tolist())
    ties = np.array([conf_thresh, max(0.15, conf_thresh - 0.3), conf_thresh + 0.1], np.float32)
    hidden = np.zeros(n_obj, np.int64)
    frames = []
    warps = np.zeros((n_frames, 2, 3), dtype=np.float64)
    warps[:, 0, 0] = warps[:, 1, 1] = 1.0
    cam = np.zeros(2)
    for f in range(n_frames):
        cx += vx
        cy += vy
        bx = (cx < 60) | (cx > img - 60)
        by = (cy < 60) | (cy > img - 60)
        vx[bx] = -vx[bx]
        vy[by] = -vy[by]
        if warp_sigma > 0:
            t = rng.normal(0, warp_sigma, 2)
            r, s = rng.normal(0, 5e-4, 2)
            warps[f] = [[1 + s, -r, t[0]], [r, 1 + s, t[1]]]
            cam += t
        alive = (born <= f) & (f < died)
        start = alive & (hidden == 0) & (rng.uniform(0, 1, n_obj) < 0.03)
        hidden[start] = rng.integers(2, 46, int(start.sum()))
        seen = alive & (hidden == 0)
        hidden[hidden > 0] -= 1
        jit = rng.normal(0, 1, (n_obj, 4))
        score = np.clip(base_score + rng.normal(0, 0.1, n_obj), 0.01, 0.99).astype(np.float32)
        tie = rng.uniform(0, 1, n_obj) < 0.05
        score[tie] = ties[rng.integers(0, 3, n_obj)[tie]]
        box = np.stack([cx - w / 2 + jit[:, 0] + cam[0], cy - h / 2 + jit[:, 1] + cam[1],
                        cx + w / 2 + jit[:, 2] + cam[0], cy + h / 2 + jit[:, 3] + cam[1]], 1)
        box = np.round(np.clip(box, 0, img))
        box[n_base:, :2] += 0.25
        ok = seen & ((box[:, 2] - box[:, 0]) >= 4) & ((box[:, 3] - box[:, 1]) >= 4)
        if f in empty:
            ok[:] = False
        d = np.concatenate([box[ok], score[ok, None], cls[ok, None]], 1).astype(np.float32)
        order = np.argsort(-d[:, 4], kind="stable")
        frames.append(np.ascontiguousarray(d[order]))
    return frames, warps


def stream_digest(frames):
    """sha1 of the raw bytes: stored with golden fixtures to detect generator drift."""
    hsh = hashlib.sha1()
    for f in frames:
        hsh.update(np.ascontiguousarray(f, dtype=np.float32).tobytes())
    return hsh.hexdigest()


def pack_frames(frames, max_dets=None):
    """List of ragged (n_i,6) arrays -> (dets (F, D, 6) float32 zero padded, counts (F,) int32)."""
    d = max(len(f) for f in frames) if max_dets is None else max_dets
    out = np.zeros((len(frames), d, 6), dtype=np.float32)
    cnt = np.zeros(len(frames), dtype=np.int32)
    for i, f in enumerate(frames):
        n = min(len(f), d)
        out[i, :n] = f[:n]
        cnt[i] = n
    return out, cnt


def textured_frame(seed, height=720, width=1280, n_rect=400):
    """Seeded uint8 BGR frame with corners for the camera-motion estimator (SURVEY.md 8f row 1): smooth multi-scale noise plus
    random rectangles of random grey level and a little pixel noise.  NumPy only (the bench must not need OpenCV)."""
    rng = np.random.default_rng(seed)
    img = np.full((height, width), 128.0, dtype=np.float32)
    for s, a in ((64, 40.0), (16, 30.0), (4, 12.0)):
        n = rng.standard_normal((height // s + 2, width // s + 2)).astype(np.float32)
        up = np.kron(n, np.ones((s, s), dtype=np.float32))
        # box-smooth the blocks once so that the field is continuous
        up = (up[: height + s, : width + s][s // 2: s // 2 + height, s // 2: s // 2 + width] + up[:height, :width]) * 0.5
        img += a * up
    for _ in range(n_rect):
        x, y = int(rng.integers(0, width - 8)), int(rng.integers(0, height - 8))
        w, h = int(rng.integers(6, 60)), int(rng.integers(6, 60))
        img[y:y + h, x:x + w] += float(rng.uniform(-70, 70))
    img += rng.standard_normal((height, width)).astype(np.float32) * 2.0
    g = np.clip(img, 0, 255)
    bgr = np.stack([g * 0.9 + 10, g, g * 0.8 + 25], -1)
    return np.clip(bgr, 0, 255).astype(np.uint8)


def moved_frame(frame, angle_deg=0.0, tx=0.0, ty=0.0):
    """``frame`` rotated by ``angle_deg`` about its centre, then shifted by (tx, ty) pixels: bilinear, edge pixels repeated.  NumPy
    only; the source coordinates are floored to 1/256 px and the weights are integers, so every platform builds the same bytes."""
    h, w = frame.shape[:2]
    a = np.deg2rad(angle_deg)
    c, s = np.cos(a), np.sin(a)
    ys, xs = np.mgrid[0:h, 0:w].astype(np.float64)
    cx, cy = (w - 1) * 0.5, (h - 1) * 0.5
    dx, dy = xs - cx - tx, ys - cy - ty
    U = np.floor((c * dx + s * dy + cx) * 256.0).astype(np.int64)
    V = np.floor((-s * dx + c * dy + cy) * 256.0).astype(np.int64)
    fx, fy = U & 255, V & 255
    x0, y0 = np.clip(U >> 8, 0, w - 1), np.clip(V >> 8, 0, h - 1)
    x1, y1 = np.clip((U >> 8) + 1, 0, w - 1), np.clip((V >> 8) + 1, 0, h - 1)
    f = frame.astype(np.int64)
    fx, fy = fx[..., None], fy[..., None]
    top = (256 - fx) * f[y0, x0] + fx * f[y0, x1]
    bot = (256 - fx) * f[y1, x0] + fx * f[y1, x1]
    return (((256 - fy) * top + fy * bot + (1 << 15)) >> 16).astype(np.uint8)


def with_flat_boxes(frame, rng, xywh=False):
    """The frame's detections plus boxes the tracker ignores (zero height, a point, a NaN box; with the xywh Kalman filter also zero width),
    high and low scores, inserted at random places; the frame's own detections keep their order."""
    src = frame[rng.choice(len(frame), 4)].astype(np.float32)
    bad = src.copy()
    bad[0, 3] = bad[0, 1]                                   # zero height (a box clipped flat against the top / bottom edge)
    bad[1, 2], bad[1, 3] = bad[1, 0], bad[1, 1]             # a point
    bad[2, :4] = np.nan
    bad[3, 3] = bad[3, 1]
    if xywh:
        bad[3, 3], bad[3, 2] = bad[3, 1] + 20.0, bad[3, 0]   # zero width: no noise scale for x / w under xywh
    bad[:, 4] = np.array([0.9, 0.8, 0.9, 0.3], np.float32)
    out = frame.astype(np.float32)
    for row in bad:
        out = np.insert(out, int(rng.integers(0, len(out) + 1)), row, axis=0)
    return out


def with_zero_width(frame, rng, frac=0.15):
    """A copy of the frame with a fraction of its boxes flattened to zero width (x2 = x1, the height kept): what scale_coords' clip
    makes of a box wholly beyond the left or right image edge.  The reference tracks such boxes (xyah filter: aspect ratio 0)."""
    out = np.array(frame, dtype=np.float32, copy=True)
    sel = rng.random(len(out)) < frac
    out[sel, 2] = out[sel, 0]
    return out


def zero_width_stream(seed, n_frames, n_obj):
    """make_stream(seed, ...) with every frame passed through with_zero_width (generator seeded with the same seed)."""
    frames, _ = make_stream(seed, n_frames, n_obj)
    rng = np.random.default_rng(seed)
    return [with_zero_width(f, rng) for f in frames]
