"""TEST INFRASTRUCTURE: NumPy restatements and runners for the multi-sequence ReID kernels of csrc/b2t_reid.cu (the crop list built
from the NMS output, the segmented batch-statistics BatchNorm, the row-mapped pooling), shared by the GPU tier
(tests/test_gpu_reid_pipeline.py) and the CPU tier (tests/test_hostsim_reid_pipeline.py).  `be` moves arrays to the kernels' memory
(reid_kernel_ref.NumpyMem for the host simulator, a torch-backed one on the GPU)."""
import numpy as np

import reid_kernel_ref as K

OVERFLOW, ZERO_SIZE, NEGATIVE = 1, 2, 4          # B2T_REID_* (include/b200track.h)


def crop_list_ref(dets, cnt, conf_thresh, H, W, cap):
    """The reference's det_high rows per sequence (botsort.py:339-346: score >= det_thresh in float32, row order) and their crops
    ori_img[int(y1):int(y2), int(x1):int(x2)] as descriptors into the (S, H, W, 3) buffer.  Returns crops (cap, 4), offsets (S + 1),
    rowmap (cap), status (S + 1) as b2t_reid_crops_from_dets writes them."""
    S, dmax = dets.shape[:2]
    thr = np.float32(conf_thresh)
    descs, rowmap, status = [], [], [0] * (S + 1)
    offsets = []
    total = 0
    for s in range(S):
        offsets.append(min(total, cap))
        for i in range(min(max(int(cnt[s]), 0), dmax)):
            if not dets[s, i, 4] >= thr:
                continue
            x1, y1, x2, y2 = list(map(int, dets[s, i, :4]))
            desc = (s * H * W * 3, 3 * W, 1, 1)
            if min(x1, y1, x2, y2) < 0:
                status[s] |= NEGATIVE
            else:
                x1, x2, y1, y2 = min(x1, W), min(x2, W), min(y1, H), min(y2, H)        # what the slice keeps
                if x2 - x1 < 1 or y2 - y1 < 1:
                    status[s] |= ZERO_SIZE
                else:
                    desc = (s * H * W * 3 + (y1 * W + x1) * 3, 3 * W, y2 - y1, x2 - x1)
            if total < cap:
                descs.append(desc)
                rowmap.append(s * dmax + i)
            else:
                status[s] |= OVERFLOW
            total += 1
    used = min(total, cap)
    offsets.append(used)
    status[S] = total
    pad = descs[0] if used else (0, 3 * W, 1, 1)
    crops = np.array(descs + [pad] * (cap - used), np.int64).reshape(cap, 4)
    rowmap = np.array(rowmap + [-1] * (cap - used), np.int32)
    return crops, np.array(offsets, np.int32), rowmap, np.array(status, np.int32)


def run_crop_list(lib, be, dets, cnt, conf_thresh, H, W, cap):
    S, dmax = dets.shape[:2]
    d_dets, d_cnt = be.put(np.ascontiguousarray(dets, np.float32)), be.put(np.asarray(cnt, np.int32))
    crops = be.put(np.full((cap, 4), -77, np.int64))
    offsets = be.put(np.full(S + 1, -77, np.int32))
    rowmap = be.put(np.full(cap, -77, np.int32))
    status = be.put(np.full(S + 1, -77, np.int32))
    rc = lib.b2t_reid_crops_from_dets(be.ptr(d_dets), be.ptr(d_cnt), S, dmax, float(conf_thresh), H, W, cap, be.ptr(crops), be.ptr(offsets),
                                      be.ptr(rowmap), be.ptr(status), be.stream())
    assert rc == 0, lib.b2t_detect_last_error()
    return be.get(crops), be.get(offsets), be.get(rowmap), be.get(status)


def crop_cases(H=40, W=56):
    """name -> (dets (S, dmax, 6) float32, counts, conf_thresh, cap): the edge cases of the crop list."""
    rng = np.random.default_rng(9)
    thr = 0.6

    def boxes(n, S=1):
        x1 = rng.integers(0, W - 8, (S, n)); y1 = rng.integers(0, H - 8, (S, n))
        b = np.stack([x1, y1, x1 + rng.integers(1, 12, (S, n)), y1 + rng.integers(1, 12, (S, n))], -1).astype(np.float32)
        b[..., :4] += rng.uniform(0, 0.99, b[..., :4].shape).astype(np.float32)       # int() truncates the fractions
        sc = rng.uniform(0.05, 0.95, (S, n, 1)).astype(np.float32)
        return np.concatenate([b, sc, np.zeros((S, n, 1), np.float32)], -1)
    cases = {}
    d = boxes(20, 3)
    cases["zero_detections"] = (d, [0, 0, 0], thr, 16)
    d = boxes(20, 2); d[..., 4] = 0.9
    cases["all_rows_high"] = (d, [20, 13], thr, 64)
    d = boxes(12, 2); d[0, 3, 4] = np.float32(thr); d[1, 5, 4] = np.nextafter(np.float32(thr), np.float32(0))
    cases["score_equal_to_thresh"] = (d, [12, 12], thr, 32)
    d = boxes(30, 5)
    cases["empty_sequences_between_full_ones"] = (d, [30, 0, 25, 0, 30], thr, 150)
    d = boxes(16, 3); d[..., 4] = 0.9
    cases["total_equals_cap"] = (d, [5, 0, 7], thr, 12)
    cases["total_is_cap_plus_1"] = (d, [5, 1, 7], thr, 12)
    cases["cap_1_overflow_in_a_later_sequence"] = (d, [1, 0, 3], thr, 1)
    d = boxes(6, 2); d[..., 4] = 0.9
    d[0, 2, :4] = [10.2, 5.0, 10.9, 20.0]                  # zero width after int()
    d[1, 4, :4] = [3.0, 7.0, 9.0, 7.0]                     # zero height
    cases["zero_width_and_zero_height"] = (d, [6, 6], thr, 12)
    d = boxes(6, 3); d[..., 4] = 0.9
    d[1, 1, 0] = -1.0                                      # int() -> -1: refused
    d[2, 0, 1] = -0.5                                      # int() -> 0: a valid crop
    d[0, 3, :4] = [W - 3.5, H - 2.2, W + 40.0, H + 9.0]    # right / bottom ends clipped to the frame
    cases["negative_coordinate_and_clipped_ends"] = (d, [6, 6, 6], thr, 18)
    return cases


def seg_bn_inputs(rng, seg_crops, ppc, c, dt, ratio, pad_crops=2):
    """x [(sum(seg_crops) + pad_crops) * ppc][c]: segment s has its own mean / std (so mixing the statistics shows) and offsets."""
    parts = []
    for n in seg_crops:
        x, _, _ = K.bn_inputs(rng, n * ppc, c, dt, ratio)
        parts.append(x)
    parts.append(K.round16(rng.normal(0, 1, (pad_crops * ppc, c)), dt))
    gamma = rng.uniform(0.5, 1.5, c).astype(np.float32)
    beta = rng.normal(0, 0.5, c).astype(np.float32)
    offsets = np.concatenate([[0], np.cumsum(seg_crops)]).astype(np.int32)
    return np.concatenate(parts), offsets, gamma, beta


def run_bn_segments(lib, be, x_rows, offsets, max_crops, ppc, c, gamma, beta, dt, relu, inplace, eps=1e-5):
    S = len(offsets) - 1
    nbytes = int(lib.b2t_batchnorm_segments_workspace_bytes(S, max_crops, ppc, c))
    assert nbytes > 0
    ws = be.put(np.full(nbytes // 8, np.nan, np.float64))
    d_x = be.put(x_rows)
    y = d_x if inplace else be.put(np.full(x_rows.shape, 0x7777, np.uint16))
    d_off = be.put(np.asarray(offsets, np.int32))
    d_g, d_b = be.put(gamma.astype(np.float32)), be.put(beta.astype(np.float32))
    rc = lib.b2t_batchnorm_batch_stats_segments(be.ptr(d_x), be.ptr(y), be.ptr(d_off), S, max_crops, ppc, c, be.ptr(d_g), be.ptr(d_b), eps,
                                                int(relu), be.ptr(ws), K.CODE[dt], be.stream())
    assert rc == 0, lib.b2t_detect_last_error()
    return be.get(y)


def run_pool_rows(lib, be, x, rowmap, n_rows, hw, dt):
    d_x, d_map = be.put(x), be.put(np.asarray(rowmap, np.int32))
    out = be.put(np.full((n_rows, 512), -7.0, np.float32))
    rc = lib.b2t_avgpool_l2norm_rows(be.ptr(d_x), be.ptr(out), be.ptr(d_map), len(rowmap), hw, 512, K.CODE[dt], be.stream())
    assert rc == 0, lib.b2t_detect_last_error()
    return be.get(out)


def widen_degenerate(dets, size):
    """The seeded random-init detector emits boxes that round to zero width or height at score 1.0 (the reference's own note at
    botsort.py:283, "why some bboxs has 0 area"); the reference exits on such a det_high crop, and no threshold avoids them.  Tests
    that need a stream of valid crops widen every box to at least 2 px inside the frame (size: its side, or its (height, width)),
    in place on the current stream, identically in every arm they compare."""
    h, w = (size, size) if isinstance(size, int) else size
    x1 = dets[..., 0].clamp(max=w - 2)
    y1 = dets[..., 1].clamp(max=h - 2)
    dets[..., 0] = x1
    dets[..., 1] = y1
    dets[..., 2] = dets[..., 2].maximum(x1 + 2)
    dets[..., 3] = dets[..., 3].maximum(y1 + 2)
