"""not-gpu: the multi-sequence ReID kernels of csrc/b2t_reid.cu under the host simulator (tests/hostsim): the crop list built from the
NMS output against a NumPy restatement of the reference's det_high selection and slicing, the segmented batch-statistics BatchNorm
against the unsegmented kernel run on each segment alone (bitwise) and against float64 (one 16-bit ulp), and the row-mapped pooling
against the existing pooling.  The GPU tier (tests/test_gpu_reid_pipeline.py) repeats these on the H100, where blocks run concurrently."""
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.join(os.path.dirname(__file__), "hostsim"))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from simlib import sim  # noqa: E402
import reid_kernel_ref as K  # noqa: E402
import reid_pipeline_ref as P  # noqa: E402

MEM = K.NumpyMem()
CASES = P.crop_cases()


@pytest.mark.parametrize("name", sorted(CASES))
def test_sim_crop_list_matches_numpy_restatement(name):
    dets, cnt, thr, cap = CASES[name]
    H, W = 40, 56
    got = P.run_crop_list(sim(), MEM, dets, cnt, thr, H, W, cap)
    exp = P.crop_list_ref(dets, cnt, thr, H, W, cap)
    for what, g, e in zip(("crops", "offsets", "rowmap", "status"), got, exp):
        assert np.array_equal(g, e), "%s: %s\n%s\n%s" % (name, what, g, e)


def test_sim_crop_list_case_coverage():
    """the cases exercise what they are named for"""
    H, W = 40, 56
    st = {n: P.crop_list_ref(*(CASES[n][:3] + (H, W, CASES[n][3])))[3] for n in CASES}
    assert st["zero_detections"][-1] == 0
    assert st["total_equals_cap"][-1] == 12 and not (st["total_equals_cap"][:-1] & P.OVERFLOW).any()
    assert st["total_is_cap_plus_1"][-1] == 13 and st["total_is_cap_plus_1"][2] & P.OVERFLOW and not st["total_is_cap_plus_1"][:2].any()
    assert st["zero_width_and_zero_height"][0] == P.ZERO_SIZE and st["zero_width_and_zero_height"][1] == P.ZERO_SIZE
    assert list(st["negative_coordinate_and_clipped_ends"][:3]) == [0, P.NEGATIVE, 0]
    d, cnt, thr, _ = CASES["score_equal_to_thresh"]
    crops, off, rowmap, _ = P.crop_list_ref(d, cnt, thr, H, W, 32)
    assert 3 in rowmap and 12 + 5 not in rowmap                      # >= in float32: equal passes, one float below does not


@pytest.mark.parametrize("dt", ["fp16", "bf16"])
@pytest.mark.parametrize("c,seg_crops,ppc,ratio,relu,inplace", [
    (64, [3, 0, 1, 5], 40, 1000, 1, 0),            # an empty segment, a single-crop one; 3 x 40 x 64: several stats blocks per segment
    (128, [0, 2, 0], 12, 100, 0, 1),               # empty first and last segments
    (256, [1, 4], 6, 10, 1, 1),
    (512, [2, 1, 0, 1], 4, 1000, 0, 0),
    (64, [30], 33, 0, 1, 0),                        # one segment over 2 stats blocks
])
def test_sim_batchnorm_segments_equal_each_segment_alone(dt, c, seg_crops, ppc, ratio, relu, inplace):
    rng = np.random.default_rng(c + sum(seg_crops) + ppc)
    x, off, gamma, beta = P.seg_bn_inputs(rng, seg_crops, ppc, c, dt, ratio)
    max_crops = len(x) // ppc
    y = P.run_bn_segments(sim(), MEM, x, off, max_crops, ppc, c, gamma, beta, dt, relu, inplace)
    for s in range(len(seg_crops)):
        a, b = off[s] * ppc, off[s + 1] * ppc
        if a == b:
            continue
        alone, _ = K.run_bn(sim(), MEM, x[a:b], b - a, c, gamma, beta, dt, relu, 0)
        assert np.array_equal(y[a:b], alone), "segment %d differs from the unsegmented kernel on it" % s
        K.assert_within_1ulp(y[a:b], K.bn_ref(x[a:b], dt, b - a, c, gamma, beta, 1e-5, relu), dt, "segment %d" % s)
    end = off[-1] * ppc
    tail = x[end:] if inplace else np.full_like(x[end:], 0x7777)
    assert np.array_equal(y[end:], tail), "padding rows written"


@pytest.mark.parametrize("dt", ["fp16", "bf16"])
def test_sim_pool_rows_equal_plain_pooling(dt):
    rng = np.random.default_rng(4)
    n, hw = 5, 6
    x = K.rand16(rng, (n, hw, 512), dt)
    plain = K.run_avgpool(sim(), MEM, x, n, hw, dt)
    rowmap = np.array([7, 0, -1, 3, -1], np.int32)
    got = P.run_pool_rows(sim(), MEM, x, rowmap, 9, hw, dt)
    for j, r in enumerate(rowmap):
        if r >= 0:
            assert np.array_equal(got[r], plain[j])
    untouched = sorted(set(range(9)) - set(int(r) for r in rowmap if r >= 0))
    assert (got[untouched] == -7.0).all()


def test_sim_argument_errors():
    import ctypes as C
    lib = sim()
    p = C.c_void_p(16)
    assert lib.b2t_batchnorm_segments_workspace_bytes(0, 4, 4, 64) == 0
    assert lib.b2t_batchnorm_segments_workspace_bytes(2, 0, 4, 64) == 0
    assert lib.b2t_batchnorm_segments_workspace_bytes(2, 4, 4, 24) == 0
    assert lib.b2t_batchnorm_batch_stats_segments(p, p, p, 2, 4, 4, 520, p, p, 1e-5, 0, p, 1, None) != 0
    assert lib.b2t_reid_crops_from_dets(p, p, 2, 8, 0.5, 10, 10, 0, p, p, p, p, None) != 0
    assert lib.b2t_avgpool_l2norm_rows(p, p, p, 1, 4, 256, 1, None) != 0
    assert b"512 channels" in lib.b2t_detect_last_error()
