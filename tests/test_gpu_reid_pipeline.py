"""-m gpu: appearance inside the multi-sequence TrackingPipeline on an H100.
  * the segmented batch-statistics BatchNorm through the C ABI: each segment bitwise equal to b2t_batchnorm_batch_stats on it alone,
    every allowed width, empty / single-crop / grid-cap segments, padding untouched, repeatable bits;
  * the crop list built on the device from the NMS output against the NumPy restatement of the reference's det_high slicing;
  * the segmented extractor: each sequence's features bitwise equal to ``features_from_frame`` on that sequence alone;
  * TrackingPipeline(reid=) against the same work done step by step on one stream, and against the drop-in BoTSORT with appearance,
    one tracker per sequence (the reference builds one per sequence and calls the extractor on each one's crops);
  * the error paths."""
import ctypes as C
import os
import sys

import numpy as np
import pytest

pytestmark = pytest.mark.gpu
torch = pytest.importorskip("torch")

HERE = os.path.dirname(os.path.abspath(__file__))
PKG = os.path.join(os.path.dirname(HERE), "yolov7-tracker_b200")
sys.path.insert(0, HERE)
import reid_kernel_ref as K  # noqa: E402
import reid_pipeline_ref as P  # noqa: E402
from b200track import _lib as L  # noqa: E402

WIDTHS = [8, 16, 32, 64, 128, 256, 512]          # every c with 8 <= c <= 512, c % 8 == 0 and c / 8 dividing 256
MAX_BLOCKS = 132 * 8                              # the stats grid's cap (kBnMaxBlocks)


class TorchMem:
    def put(self, a):
        a = np.ascontiguousarray(a)
        if a.dtype == np.uint16:
            a = a.view(np.int16)
        return torch.from_numpy(a.copy()).cuda()

    def ptr(self, t):
        return C.c_void_p(t.data_ptr())

    def get(self, t):
        torch.cuda.synchronize()
        a = t.cpu().numpy()
        return a.view(np.uint16) if a.dtype == np.int16 else a

    def stream(self):
        return C.c_void_p(torch.cuda.current_stream().cuda_stream)


MEM = TorchMem()


@pytest.fixture(scope="module")
def lib():
    return L.load()


# ---------------------------------------------------------------- 1. segmented BatchNorm == the unsegmented kernel per segment

@pytest.mark.parametrize("dt", ["fp16", "bf16"])
@pytest.mark.parametrize("c", WIDTHS)
def test_batchnorm_segments_bitwise_equal_each_segment_alone(lib, dt, c):
    ppc = 512
    ppb = 256 // (c // 8)
    at_cap = (MAX_BLOCKS * ppb * 16 + ppc - 1) // ppc + 1       # a segment whose own grid is the capped one
    seg_crops = [0, 1, 7, 0, at_cap, 3]
    rng = np.random.default_rng(c)
    x, off, gamma, beta = P.seg_bn_inputs(rng, seg_crops, ppc, c, dt, 1000 if c % 16 == 0 else 100)
    max_crops = len(x) // ppc
    relu = int(c % 32 == 0)
    y = P.run_bn_segments(lib, MEM, x, off, max_crops, ppc, c, gamma, beta, dt, relu, 0)
    for s in range(len(seg_crops)):
        a, b = off[s] * ppc, off[s + 1] * ppc
        if a == b:
            continue
        alone, _ = K.run_bn(lib, MEM, x[a:b], b - a, c, gamma, beta, dt, relu, 0)
        assert np.array_equal(y[a:b], alone), "c=%d segment %d (%d crops) differs from b2t_batchnorm_batch_stats on it alone" % (c, s, seg_crops[s])
    assert (y[off[-1] * ppc:] == 0x7777).all(), "padding rows written"
    yi = P.run_bn_segments(lib, MEM, x, off, max_crops, ppc, c, gamma, beta, dt, relu, 1)          # in place
    assert np.array_equal(yi[:off[-1] * ppc], y[:off[-1] * ppc]) and np.array_equal(yi[off[-1] * ppc:], x[off[-1] * ppc:])


def test_batchnorm_segments_repeatable_bits(lib):
    rng = np.random.default_rng(5)
    x, off, gamma, beta = P.seg_bn_inputs(rng, [40, 0, 1, 300], 256, 64, "fp16", 1000)
    outs = [P.run_bn_segments(lib, MEM, x, off, len(x) // 256, 256, 64, gamma, beta, "fp16", 1, 0) for _ in range(5)]
    for o in outs[1:]:
        assert np.array_equal(o, outs[0]), "segmented BatchNorm differs between identical calls"


def test_argument_errors(lib):
    p = C.c_void_p(16)
    assert lib.b2t_batchnorm_segments_workspace_bytes(0, 4, 4, 64) == 0
    assert lib.b2t_batchnorm_batch_stats_segments(p, p, p, 2, 4, 4, 24, p, p, 1e-5, 0, p, 1, None) == -1
    assert lib.b2t_reid_crops_from_dets(p, p, 2, 8, 0.5, 10, 10, 0, p, p, p, p, None) == -1
    assert lib.b2t_avgpool_l2norm_rows(p, p, p, 1, 4, 256, 1, None) == -1


# ---------------------------------------------------------------- 2. crop list

@pytest.mark.parametrize("name", sorted(P.crop_cases()))
def test_crop_list_matches_numpy_restatement(lib, name):
    dets, cnt, thr, cap = P.crop_cases()[name]
    got = P.run_crop_list(lib, MEM, dets, cnt, thr, 40, 56, cap)
    exp = P.crop_list_ref(dets, cnt, thr, 40, 56, cap)
    for what, g, e in zip(("crops", "offsets", "rowmap", "status"), got, exp):
        assert np.array_equal(g, e), "%s: %s" % (name, what)


def test_crop_list_many_rows(lib):
    """more rows than one block pass (256) per sequence, a cap in the middle of a sequence"""
    rng = np.random.default_rng(2)
    S, dmax, H, W = 4, 700, 300, 500
    x1 = rng.uniform(0, W - 40, (S, dmax)); y1 = rng.uniform(0, H - 40, (S, dmax))
    d = np.stack([x1, y1, x1 + rng.uniform(1, 40, (S, dmax)), y1 + rng.uniform(1, 40, (S, dmax)), rng.uniform(0, 1, (S, dmax)),
                  np.zeros((S, dmax))], -1).astype(np.float32)
    cnt = np.array([700, 0, 513, 257], np.int32)
    for cap in (S * dmax, 400):
        got = P.run_crop_list(lib, MEM, d, cnt, 0.3, H, W, cap)
        exp = P.crop_list_ref(d, cnt, 0.3, H, W, cap)
        for g, e in zip(got, exp):
            assert np.array_equal(g, e)


# ---------------------------------------------------------------- 3. the segmented extractor == features_from_frame per sequence

@pytest.fixture(scope="module")
def extractors():
    from oracle import reid as R
    from b200track.reid import ReidExtractor
    sd = R.seeded_state_dict(3)
    return {(dt, m): ReidExtractor(sd, dtype=getattr(torch, dt), bn_mode=m) for dt in ("float16", "bfloat16") for m in ("batch", "running")}


def _boxes(rng, n, H, W):
    x1 = rng.uniform(0, W - 30, n); y1 = rng.uniform(0, H - 50, n)
    return np.stack([x1, y1, x1 + rng.uniform(4, 120, n), y1 + rng.uniform(8, 200, n)], 1).astype(np.float32)


@pytest.mark.parametrize("S", [1, 3, 8])
@pytest.mark.parametrize("mode", ["batch", "running"])
@pytest.mark.parametrize("dt", ["float16", "bfloat16"])
def test_segmented_extractor_equals_features_from_frame(extractors, S, mode, dt):
    ext = extractors[(dt, mode)]
    rng = np.random.default_rng(S * 10 + len(mode))
    H, W = 240, 320
    frames = torch.from_numpy(rng.integers(0, 256, (S, H, W, 3), dtype=np.uint8)).cuda()
    counts = [int(v) for v in rng.integers(1, 40, S)]
    if S > 1:
        counts[1] = 0                                               # an empty sequence between full ones
    if S == 8:
        counts[7] = 0; counts[3] = 1
    tl = [_boxes(rng, n, H, W) for n in counts]
    total = sum(counts)
    for cap in (None, total):
        got = ext.features_segments(frames, tl, cap=cap)
        for s in range(S):
            if counts[s] == 0:
                assert got[s].shape == (0, 512)
                continue
            alone = ext.features_from_frame(frames[s], tl[s])
            assert torch.equal(got[s], alone), "S=%d %s %s cap=%s: sequence %d differs from features_from_frame alone" % (S, mode, dt, cap, s)
    if mode == "batch" and S > 1:
        mixed = ext.features_from_frame(frames[0], np.concatenate([tl[0], tl[2]]))[:counts[0]]
        assert not torch.equal(mixed, got[0]), "statistics of two sequences mixed give the same features: the test shows nothing"


def test_segmented_extractor_refuses_bad_boxes(extractors):
    ext = extractors[("float16", "batch")]
    frames = torch.zeros((2, 64, 64, 3), dtype=torch.uint8, device="cuda")
    ok = np.array([[1, 1, 20, 30]], np.float32)
    with pytest.raises(L.B2TError, match="sequence 1: .*zero size"):
        ext.features_segments(frames, [ok, np.array([[5, 5, 5.9, 30]], np.float32)])
    with pytest.raises(L.B2TError, match="sequence 0: .*negative"):
        ext.features_segments(frames, [np.array([[-1, 5, 10, 30]], np.float32), ok])
    with pytest.raises(L.B2TError, match="exceed reid_cap = 1"):
        ext.features_segments(frames, [ok, ok], cap=1)


# ---------------------------------------------------------------- 4 / 5. TrackingPipeline(reid=)

# (detector canvas (H, W), source frames (h, w)) that are not the identity: 720p into 384 x 640 (gain 1/2, pad 12) and 360 x 640 into
# 384 x 640 (gain 1, pad 12) -- pipeline rows are in source-frame pixels, as tracker/track.py:240 produces them
LETTERBOXED = [((384, 640), (720, 1280)), ((384, 640), (360, 640))]
LETTERBOXED_IDS = ["720p_in_384x640", "360x640_in_384x640"]


def _scenario(S=3, n=6, hw=(256, 256)):
    from b200track.synth import textured_frame
    base = np.stack([textured_frame(300 + s, hw[0], hw[1], n_rect=300) for s in range(S)])
    return [torch.from_numpy(np.ascontiguousarray(np.roll(base, (3 * k, -2 * k), axis=(1, 2)))).pin_memory() for k in range(n)]


def _detector(sd, S, canvas=(256, 256), src=(256, 256)):
    from b200track.detector import DetectorW6
    det = DetectorW6(sd, batch=S, img_size=canvas, use_graph=False, autotune=False)
    det.set_source_frames(src)
    return det


def _reference_rows(det, f):
    """the reference's way (tracker/track.py:143-145, 239-240): letterbox the frames, detect on the canvas without
    post-processing, then scale_coords(...).round() back to the source frame with the drop-in utils.general.  Also leaves the
    frames in det.src_u8.  Returns (rows (S, dmax, 6) float32, counts (S,) int32) device tensors."""
    from b200track.preprocess import Letterbox
    from utils.general import scale_coords
    det.src_u8.copy_(f)
    img, _ = Letterbox(max(det.H, det.W), 64)(det.src_u8)
    assert tuple(img.shape[2:]) == (det.H, det.W)
    out, cnt = det.detect(img, post=False)
    rows = out.clone()
    for s in range(det.B):
        rows[s, :, :4] = scale_coords((det.H, det.W), rows[s, :, :4], det.src_hw).round()
    return rows, cnt.clone()


def _pick_thresh(det, frames):
    """conf_thresh 0.2 unless a frame has no det_high row then (the boxes widened as in the runs below, so none is refused)"""
    h, w = det.src_hw
    for thr in (0.2, 0.1, 0.05):
        ok = True
        for f in frames:
            rows, cnt = _reference_rows(det, f)
            P.widen_degenerate(rows, (h, w))
            torch.cuda.synchronize()
            d, c = rows.cpu().numpy(), cnt.cpu().numpy()
            st = P.crop_list_ref(d, c, thr, h, w, d.shape[0] * d.shape[1])[3]
            assert not st[:-1].any()
            ok = ok and st[-1] >= 1
        if ok:
            return thr
    pytest.fail("no det_high rows on this stream")


def _widened_pipeline(pipe, size=(256, 256)):
    """every detector's NMS output widened inside the source frame on the tracker stream before the crop list (and so before GMC
    and the step)"""
    cut = pipe.reid_net.cut

    def widened_cut(fr, d, cnt, t):
        P.widen_degenerate(d, size)
        return cut(fr, d, cnt, t)
    pipe.reid_net.cut = widened_cut
    return pipe


def _run_pipeline(pipe, frames, S):
    got = []
    for f in frames:
        r = pipe.step(f)
        if r is not None:
            got.append([r[0][s, :int(r[1][s, L.STAT_NOUT])].clone() for s in range(S)])
    r = pipe.flush()
    got.append([r[0][s, :int(r[1][s, L.STAT_NOUT])].clone() for s in range(S)])
    return got


def _stepwise(det, eng, ext, frames, S, gmc=None):
    """letterbox -> detect -> NMS -> scale_coords to the source frame (the reference's way, not the pipeline's NMS graph) -> [GMC on
    the source frame] -> per-sequence features_from_frame of the det_high rows -> scatter -> step_device(feats=), one stream"""
    thr = np.float32(eng.cfg.conf_thresh)
    out = torch.zeros((S, eng.cap, L.OUT_COLS), dtype=torch.float64, device="cuda")
    stat = torch.zeros((S, L.STAT_WORDS), dtype=torch.int32, device="cuda")
    feats = torch.zeros((S, eng.dmax, 512), dtype=torch.float32, device="cuda")
    exp, dets = [], []
    for f in frames:
        rows, rcnt = _reference_rows(det, f)
        P.widen_degenerate(rows, det.src_hw)
        w = None
        if gmc is not None:
            w23, _ = gmc.estimate(det.src_u8, rows, rcnt, det_thresh=float(eng.cfg.conf_thresh))
            w = w23.view(S, 6)
        d = rows.cpu().numpy(); cnt = rcnt.cpu().numpy()
        dets.append([d[s, :cnt[s]].copy() for s in range(S)])
        for s in range(S):
            hi = np.nonzero(d[s, :cnt[s], 4] >= thr)[0]
            if len(hi):
                feats[s, torch.from_numpy(hi).cuda()] = ext.features_from_frame(det.src_u8[s], d[s, hi, :4])
        eng.step_device(rows, rcnt, out, stat, warps=w, feats=feats)
        torch.cuda.synchronize()
        assert int(stat[:, L.STAT_ERR].max()) == 0
        exp.append([out[s, :int(stat[s, L.STAT_NOUT])].cpu().clone() for s in range(S)])
    return exp, dets


def _assert_rows_equal(got, exp, S):
    assert len(got) == len(exp)
    rows = 0
    for k, (a, b) in enumerate(zip(got, exp)):
        for s in range(S):
            assert a[s].shape == b[s].shape and torch.equal(a[s], b[s]), "frame %d sequence %d" % (k, s)
            rows += a[s].shape[0]
    assert rows > 0


@pytest.fixture(scope="module")
def w6_sd():
    from b200track.w6 import calibrated_state_dict
    return calibrated_state_dict(0, 256, "cuda")


def _engine(S, dmax, thr, use_gmc):
    from b200track.engine import TrackEngine
    return TrackEngine("botsort", n_seq=S, cap=1152, dmax=dmax, feat_dim=512, conf_thresh=thr, use_gmc=use_gmc)


def test_pipeline_reid_equals_stepwise_and_dropin(w6_sd, extractors):
    """one detector, no GMC: pipeline rows == stepwise rows (bitwise), and == the drop-in BoTSORT(use_apperance_model=True) run per
    sequence on the same NMS rows and frames (ids up to a per-sequence offset, boxes within 1e-9)"""
    _reid_equals_stepwise_and_dropin(w6_sd, extractors, (256, 256), (256, 256))


@pytest.mark.parametrize("geo", LETTERBOXED, ids=LETTERBOXED_IDS)
def test_pipeline_reid_equals_stepwise_and_dropin_letterboxed(w6_sd, extractors, geo):
    _reid_equals_stepwise_and_dropin(w6_sd, extractors, *geo)


def _reid_equals_stepwise_and_dropin(w6_sd, extractors, canvas, src):
    from b200track.pipeline import TrackingPipeline
    S = 3
    frames = _scenario(S, hw=src)
    ext = extractors[("float16", "batch")]
    det = _detector(w6_sd, S, canvas, src)
    thr = _pick_thresh(det, frames)
    pipe = _widened_pipeline(TrackingPipeline(det, _engine(S, det.max_det, thr, False), out_rows=1152, reid=ext), src)
    got = _run_pipeline(pipe, frames, S)
    assert int(pipe.h_rstat[0][S]) + int(pipe.h_rstat[1][S]) > 0, "no det_high crops: the test shows nothing"
    exp, dets = _stepwise(_detector(w6_sd, S, canvas, src), _engine(S, det.max_det, thr, False), ext, frames, S)
    _assert_rows_equal(got, exp, S)
    # ---- the drop-in, one tracker per sequence (reference tracker/track.py:123,132), fed the same NMS rows and frames
    saved = {k: sys.modules.pop(k) for k in list(sys.modules) if k in ("basetrack", "botsort", "matching", "kalman_filter")}
    sys.path.insert(0, os.path.join(PKG, "tracker"))
    try:
        from basetrack import BaseTrack
        from botsort import BoTSORT

        class Opts:
            conf_thresh = thr; track_buffer = 30; kalman_format = "botsort"; img_size = 256; iou_thresh = 0.5
            reid_model_path = ""; dhn_path = ""
        compared = 0
        for s in range(S):
            BaseTrack._count = 0
            trk = BoTSORT(Opts(), use_GMC=False)
            trk.use_apperance_model = True
            trk.reid_model = ext
            offset = None
            for k, f in enumerate(frames):
                out = trk.update(dets[k][s].copy(), f[s].numpy())
                ids = np.array(sorted(int(t.track_id) for t in out), np.int64)
                mine = got[k][s].numpy()
                order = np.argsort(mine[:, 0], kind="stable")
                pid = mine[order, 0].astype(np.int64)
                assert len(ids) == len(pid), "frame %d sequence %d" % (k, s)
                if len(ids):
                    offset = ids[0] - pid[0] if offset is None else offset
                    assert np.array_equal(ids - pid, np.full_like(ids, offset)), "frame %d sequence %d" % (k, s)
                    box = {int(t.track_id): t.tlwh for t in out}
                    np.testing.assert_allclose(np.array([box[int(i)] for i in ids]), mine[order, 1:5], rtol=0, atol=1e-9)
                    compared += len(ids)
        assert compared > 0
    finally:
        sys.path.remove(os.path.join(PKG, "tracker"))
        for k in ("basetrack", "botsort", "matching", "kalman_filter"):
            sys.modules.pop(k, None)
        sys.modules.update(saved)


def test_pipeline_reid_twins_with_gpu_gmc_equals_stepwise(w6_sd, extractors):
    _reid_twins_with_gmc(w6_sd, extractors, (256, 256), (256, 256))


@pytest.mark.parametrize("geo", LETTERBOXED, ids=LETTERBOXED_IDS)
def test_pipeline_reid_twins_with_gpu_gmc_equals_stepwise_letterboxed(w6_sd, extractors, geo):
    """twin detectors with GMC on the source frame, at a source size that is not the canvas"""
    _reid_twins_with_gmc(w6_sd, extractors, *geo)


def _reid_twins_with_gmc(w6_sd, extractors, canvas, src):
    from b200track.gmc import GmcEstimator
    from b200track.pipeline import TrackingPipeline
    S = 2
    frames = _scenario(S, hw=src)
    ext = extractors[("bfloat16", "batch")]
    dets = [_detector(w6_sd, S, canvas, src), _detector(w6_sd, S, canvas, src)]
    thr = _pick_thresh(dets[0], frames)
    gmc = GmcEstimator(S, src[0], src[1], 2, max_kp=4096)
    pipe = _widened_pipeline(TrackingPipeline(dets, _engine(S, dets[0].max_det, thr, True), out_rows=1152, gmc=gmc, reid=ext), src)
    got = _run_pipeline(pipe, frames, S)
    warps_pipe = gmc.warps.cpu().numpy().copy()
    gmc2 = GmcEstimator(S, src[0], src[1], 2, max_kp=4096)
    exp, _ = _stepwise(_detector(w6_sd, S, canvas, src), _engine(S, dets[0].max_det, thr, True), ext, frames, S, gmc=gmc2)
    _assert_rows_equal(got, exp, S)
    np.testing.assert_array_equal(warps_pipe, gmc2.warps.cpu().numpy())


# ---------------------------------------------------------------- 6. error paths

def test_pipeline_reid_errors(w6_sd, extractors):
    from b200track.engine import TrackEngine
    from b200track.pipeline import TrackingPipeline
    S = 2
    frames = _scenario(S, n=2)
    ext = extractors[("float16", "running")]
    det = _detector(w6_sd, S)
    thr = _pick_thresh(det, frames)
    with pytest.raises(L.B2TError, match="BoT-SORT with feat_dim=512"):
        TrackingPipeline(det, TrackEngine("botsort", n_seq=S, cap=1152, dmax=det.max_det), reid=ext)
    with pytest.raises(L.B2TError, match="BoT-SORT with feat_dim=512"):
        TrackingPipeline(det, TrackEngine("bytetrack", n_seq=S, cap=1152, dmax=det.max_det), reid=ext)
    with pytest.raises(L.B2TError, match="reid_cap must be >= 1"):
        TrackingPipeline(det, _engine(S, det.max_det, thr, False), reid=ext, reid_cap=0)
    pipe = TrackingPipeline(det, _engine(S, det.max_det, thr, False), out_rows=1152, reid=ext)
    with pytest.raises(L.B2TError, match="uint8"):
        pipe.step(torch.zeros((S, 3, 256, 256), dtype=torch.float32, device="cuda"))
    # a cap below the crops of a frame
    pipe = _widened_pipeline(TrackingPipeline(det, _engine(S, det.max_det, thr, False), out_rows=1152, reid=ext, reid_cap=1))
    pipe.step(frames[0])
    with pytest.raises(L.B2TError, match="exceed reid_cap = 1"):
        pipe.flush()
    # a zero-size det_high box (row 0 of sequence 0 made zero-width and high-scoring on the tracker stream, before the crop list)
    pipe = TrackingPipeline(det, _engine(S, det.max_det, thr, False), out_rows=1152, reid=ext)
    cut = pipe.reid_net.cut

    def bad_cut(fr, d, cnt, t):
        P.widen_degenerate(d, 256)
        d[0, 0, 2].copy_(d[0, 0, 0])
        d[0, 0, 4].fill_(1.0)
        cnt[0:1].clamp_(min=1)
        return cut(fr, d, cnt, t)
    pipe.reid_net.cut = bad_cut
    pipe.step(frames[0])
    with pytest.raises(L.B2TError, match="sequence 0: .*zero size"):
        pipe.flush()
