"""Drop-in for the reference's ``tracker/matching.py``.

GPU-backed (libb200track.so):
  ious / iou_distance          reference :44-82   -> b2t_iou_cost   ("+1" IoU, float64)
  linear_assignment            reference :30-41   -> b2t_lap_solve  (exact, lap.lapjv(extend_cost, cost_limit) semantics)
  buffered_iou_distance        reference :391-407 -> b2t_iou_cost
  fuse_motion                  reference :202-213 -> b2t_kalman_gating
  matching_cascade             reference :216-279 -> linear_assignment per level
Appearance costs (cosine / euclidean GEMMs, out of the section-8 hot path) run on the GPU through torch;
the UAVMOT structure costs are not provided (NotImplementedError).
"""
import numpy as np

import _b2t_path  # noqa: F401
import kalman_filter
from b200track import _lib as L
from b200track import engine as _eng

import torch  # noqa: E402


def merge_matches(m1, m2, shape):
    o, p, q = shape
    a = np.zeros((o, p)); b = np.zeros((p, q))
    m1 = np.asarray(m1).reshape(-1, 2); m2 = np.asarray(m2).reshape(-1, 2)
    a[m1[:, 0], m1[:, 1]] = 1
    b[m2[:, 0], m2[:, 1]] = 1
    rows, cols = np.nonzero(a @ b)
    match = list(zip(rows, cols))
    return match, tuple(set(range(o)) - set(rows.tolist())), tuple(set(range(q)) - set(cols.tolist()))


def linear_assignment(cost_matrix, thresh):
    cost_matrix = np.asarray(cost_matrix)
    if cost_matrix.size == 0:
        return np.empty((0, 2), dtype=int), tuple(range(cost_matrix.shape[0])), tuple(range(cost_matrix.shape[1]))
    ops = _eng.ops()
    c = ops.dev(cost_matrix.astype(np.float64), torch.float64)
    x, y = ops.lap_solve(L.F64, c, float(thresh))
    x = x.cpu().numpy().astype(np.int64); y = y.cpu().numpy().astype(np.int64)
    rows = np.nonzero(x >= 0)[0]
    matches = np.stack([rows, x[rows]], 1) if len(rows) else np.asarray([])
    return matches, np.where(x < 0)[0], np.where(y < 0)[0]


def ious(atlbrs, btlbrs):
    n, m = len(atlbrs), len(btlbrs)
    if n * m == 0:
        return np.zeros((n, m), dtype=np.float64)
    ops = _eng.ops()
    a = ops.dev(np.ascontiguousarray(atlbrs, dtype=np.float64).reshape(n, 4), torch.float64)
    b = ops.dev(np.ascontiguousarray(btlbrs, dtype=np.float64).reshape(m, 4), torch.float64)
    return ops.iou_cost(L.F64, a, b, as_distance=False).cpu().numpy()


def iou_distance(atracks, btracks):
    if (len(atracks) > 0 and isinstance(atracks[0], np.ndarray)) or (len(btracks) > 0 and isinstance(btracks[0], np.ndarray)):
        atlbrs, btlbrs = atracks, btracks
    else:
        atlbrs = [t.tlbr for t in atracks]
        btlbrs = [t.tlbr for t in btracks]
    return 1 - ious(atlbrs, btlbrs)


def buffered_iou_distance(atracks, btracks, level=1):
    assert level in [1, 2], 'level must be 1 or 2'
    if level == 1:
        atlbrs = [t.tlwh2tlbr(t.motion_state1) for t in atracks]
        btlbrs = [d.tlwh2tlbr(d.buffer_bbox1) for d in btracks]
    else:
        atlbrs = [t.tlwh2tlbr(t.motion_state2) for t in atracks]
        btlbrs = [d.tlwh2tlbr(d.buffer_bbox2) for d in btracks]
    return 1 - ious(atlbrs, btlbrs)


_cos_gemm = None


def cal_cosine_distance(mat1, mat2):
    """normalize(mat1) @ normalize(mat2).T (reference :165-178) on the wgmma conv kernel as a split-fp16 GEMM
    (b200track/gemm.py): float64-level results (~1e-6) from the tensor cores."""
    global _cos_gemm
    ops = _eng.ops()
    a = ops.dev(np.asarray(mat1, dtype=np.float64), torch.float64)
    b = ops.dev(np.asarray(mat2, dtype=np.float64), torch.float64)
    if a.shape[0] == 0 or b.shape[0] == 0:
        return np.zeros((a.shape[0], b.shape[0]))
    if _cos_gemm is None:
        from b200track.gemm import CosineGemm
        _cos_gemm = CosineGemm(device=ops.device, dim=a.shape[1])
    return _cos_gemm.cosine_similarity(a, b).double().cpu().numpy()


def cal_eculidian_distance(mat1, mat2):
    if len(mat1) == 0 or len(mat2) == 0:
        return np.zeros((len(mat1), len(mat2)))
    ops = _eng.ops()
    a = ops.dev(np.asarray(mat1, dtype=np.float64), torch.float64)
    b = ops.dev(np.asarray(mat2, dtype=np.float64), torch.float64)
    d = (-2 * a @ b.T + (a * a).sum(1)[:, None] + (b * b).sum(1)[None, :]).clamp_(min=0)
    return np.minimum(0.0, d.min(dim=0).values.cpu().numpy())     # sic: the reference returns min(0, .)


def embedding_distance(tracks, detections, metric='cosine'):
    cost = np.zeros((len(tracks), len(detections)), dtype=np.float64)
    if cost.size == 0:
        return cost
    det_f = np.asarray([t.features[-1] for t in detections], dtype=np.float64)
    trk_f = np.asarray([t.features[-1] for t in tracks], dtype=np.float64)
    if metric == 'cosine':
        return 1. - cal_cosine_distance(trk_f, det_f)
    if metric == 'euclidean':
        ops = _eng.ops()
        return torch.cdist(ops.dev(trk_f, torch.float64), ops.dev(det_f, torch.float64)).clamp_(min=0).cpu().numpy()
    raise NotImplementedError


def nearest_embedding_distance(tracks, detections, metric='cosine'):
    cost = np.zeros((len(tracks), len(detections)))
    det_f = np.asarray([d.features[-1] for d in detections])
    for row, track in enumerate(tracks):
        cost[row, :] = (1. - cal_cosine_distance(np.asarray(track.features), det_f)).min(axis=0)
    return cost


def ecu_iou_distance(tracks, detections, img0_shape):
    cost = np.zeros((len(tracks), len(detections)), dtype=np.float64)
    if cost.size == 0:
        return cost
    det = np.asarray([d.tlwh for d in detections], dtype=np.float64)
    trk = np.asarray([t.tlwh for t in tracks], dtype=np.float64)
    dc = det[:, :2] + 0.5 * det[:, 2:]
    tc = trk[:, :2] + 0.5 * trk[:, 2:]
    ecu = np.sqrt(((tc[:, None, :] - dc[None, :, :]) ** 2).sum(-1))
    ecu = 1. - np.exp(-5 * ecu / float((img0_shape[0] ** 2 + img0_shape[1] ** 2) ** 0.5))
    return 0.5 * (ecu + iou_distance(tracks, detections))


def fuse_motion(kf, cost_matrix, tracks, detections, only_position=False, lambda_=0.98):
    if cost_matrix.size == 0:
        return cost_matrix
    gate = kalman_filter.chi2inv95[2 if only_position else 4]
    meas = np.asarray([d.to_xyah() for d in detections])
    for row, track in enumerate(tracks):
        g = kf.gating_distance(track.mean, track.covariance, meas, only_position, metric='maha')
        cost_matrix[row, g > gate] = np.inf
        cost_matrix[row] = lambda_ * cost_matrix[row] + (1 - lambda_) * g
    return cost_matrix


def matching_cascade(distance_metric, matching_thresh, cascade_depth, tracks, detections,
                     track_indices=None, detection_indices=None):
    if track_indices is None:
        track_indices = list(range(len(tracks)))
    if detection_indices is None:
        detection_indices = list(range(len(detections)))
    todo, matches = detection_indices, []
    for level in range(cascade_depth):
        if not len(todo):
            break
        level_tracks = [k for k in track_indices if tracks[k].time_since_update == 1 + level]
        if not len(level_tracks):
            continue
        cost = distance_metric([tracks[i] for i in level_tracks], [detections[i] for i in todo])
        pairs, _, um_cols = linear_assignment(cost, matching_thresh)
        for r, c in pairs:
            matches.append((level_tracks[r], todo[c]))
        todo = [todo[c] for c in um_cols]
    unmatched_tracks = list(set(track_indices) - set(k for k, _ in matches))
    return matches, unmatched_tracks, todo


def _uavmot_unavailable(*a, **k):
    raise NotImplementedError("UAVMOT structure costs (reference matching.py:284-389) are outside the accelerated "
                              "detect->NMS->associate path (SURVEY.md section 2.1 row 3) and are not provided")


local_relation_fuse_motion = structure_similarity_distance = structure_representation = _uavmot_unavailable


def angle(v1, v2):
    import math
    a1 = int(math.atan2(v1[1], v1[0]) * 180 / math.pi)
    a2 = int(math.atan2(v2[1], v2[0]) * 180 / math.pi)
    if a1 * a2 >= 0:
        return abs(a1 - a2)
    inc = abs(a1) + abs(a2)
    return 360 - inc if inc > 180 else inc
