"""-m gpu: BoT-SORT with appearance features through the fused step (b2t_tracker_step_feat) and the drop-in BoTSORT, against the
reference-pinned golden (tests/golden/loop_botsort_reid.npz) and the oracle (tests/reid_track_oracle.py)."""
import ctypes as C
import os
import sys

import numpy as np
import pytest

pytestmark = pytest.mark.gpu
torch = pytest.importorskip("torch")

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
PKG = os.path.join(ROOT, "yolov7-tracker_b200")
sys.path.insert(0, HERE)
from b200track import _lib as L  # noqa: E402
from b200track.synth import make_reid_stream  # noqa: E402
from reid_track_oracle import ReidBotsortOracle  # noqa: E402

GOLDEN = os.path.join(HERE, "golden")
EINVAL = -1


def _golden():
    g = np.load(os.path.join(GOLDEN, "loop_botsort_reid.npz"))
    seed, n_obj, n_frames, dim = [int(v) for v in g["cfg"]]
    frames, feats, warps = make_reid_stream(seed, n_frames, n_obj, dim)
    return g, frames, feats, warps


def _step(eng, frames, feats, warps):
    dev = eng.device
    return eng.step_cuda_dets([torch.from_numpy(f).to(dev) for f in frames], warps=np.stack(warps).reshape(len(frames), 6),
                              feats_list=[torch.from_numpy(x).to(dev) for x in feats])


@pytest.mark.parametrize("dtype", ["f64", "f32"])
def test_step_feat_vs_reference_golden(dtype):
    """fp64: ids exact, tlwh 1e-9, smoothed features 1e-6 on every stored frame; fp32: ids exact, tlwh 1e-4 relative."""
    from b200track.engine import TrackEngine
    g, frames, feats, warps = _golden()
    dim = int(g["cfg"][3])
    eng = TrackEngine("botsort", n_seq=1, dtype=dtype, cap=256, dmax=256, feat_dim=dim)
    off = np.concatenate([[0], np.cumsum(g["count"])])
    fk = {int(f): i for i, f in enumerate(g["feat_frames"])}
    foff = np.concatenate([[0], np.cumsum(g["count"][g["feat_frames"]])])
    napp = nlow = 0
    for i in range(len(frames)):
        got = _step(eng, [frames[i]], [feats[i]], [warps[i]])[0]
        napp += int(eng.np_stat[0, L.STAT_NAPP]); nlow += int(eng.np_stat[0, L.STAT_NAPPLOW])
        assert np.array_equal(got[:, 0].astype(np.int64), g["ids"][off[i]:off[i + 1]]), "%s: ids differ at frame %d" % (dtype, i + 1)
        if dtype == "f64":
            np.testing.assert_allclose(got[:, 1:5], g["tlwh"][off[i]:off[i + 1]], rtol=1e-9, atol=1e-9)
            if i in fk:
                exp = g["feats"][foff[fk[i]]:foff[fk[i] + 1]]
                f = np.stack([eng.read_feature(0, s) for s in got[:, 7]]) if len(got) else exp
                np.testing.assert_allclose(f, exp, rtol=0, atol=1e-6)
        else:
            np.testing.assert_allclose(got[:, 1:5], g["tlwh"][off[i]:off[i + 1]], rtol=1e-4, atol=2e-2)
    assert napp > 0 and 0 < nlow <= napp
    print("%s: %d appearance pairs, %d lowered by the appearance cost" % (dtype, napp, nlow))


@pytest.mark.parametrize("dim", [512, 128])
def test_step_feat_four_sequences_vs_oracle(dim):
    """Four fresh sequences of about 250 detections per frame in one launch: ids exact against the oracle."""
    from b200track.engine import TrackEngine
    S, n_frames = 4, 24
    streams = [make_reid_stream(100 + s, n_frames, 280, dim) for s in range(S)]
    eng = TrackEngine("botsort", n_seq=S, cap=1024, dmax=512, feat_dim=dim)
    orcs = [ReidBotsortOracle() for _ in range(S)]
    ndet = []
    for i in range(n_frames):
        got = _step(eng, [st[0][i] for st in streams], [st[1][i] for st in streams], [st[2][i] for st in streams])
        assert int(eng.np_stat[:, L.STAT_ERR].max()) == 0
        for s in range(S):
            exp = orcs[s].update(streams[s][0][i], streams[s][2][i], feats=streams[s][1][i])
            assert [int(v) for v in got[s][:, 0]] == [e[0] for e in exp], "dim %d seq %d frame %d" % (dim, s, i + 1)
            ndet.append(len(streams[s][0][i]))
    assert 200 <= np.mean(ndet) <= 300
    assert int(eng.np_stat[:, L.STAT_NAPP].sum()) > 0


def test_feat_dim_zero_is_the_iou_tracker():
    """feat_dim = 0: same state size and the same outputs as before the feature path existed; the entry points do not mix."""
    from b200track.engine import TrackEngine
    frames, feats, warps = make_reid_stream(7, 16, 80, 64)
    a = TrackEngine("botsort", cap=256, dmax=256)
    b = TrackEngine("botsort", cap=256, dmax=256, feat_dim=0, theta_iou=0.3, theta_emb=0.1)
    assert a.lib.b2t_tracker_state_bytes(C.byref(a.cfg)) == b.lib.b2t_tracker_state_bytes(C.byref(b.cfg))
    for i, f in enumerate(frames):
        ra = a.step([f], warps=warps[i].reshape(1, 6))[0]
        rb = b.step_cuda_dets([torch.from_numpy(f).cuda()], warps=warps[i].reshape(1, 6))[0]
        assert np.array_equal(ra, rb)
        assert int(b.np_stat[0, L.STAT_NAPP]) == 0
    lib = a.lib
    c = TrackEngine("botsort", cap=256, dmax=256, feat_dim=64)
    d = torch.zeros((1, 256, 6), device="cuda"); n = torch.zeros(1, dtype=torch.int32, device="cuda")
    fe = torch.zeros((1, 256, 64), device="cuda")
    out = torch.zeros((1, 256, 8), dtype=torch.float64, device="cuda"); st = torch.zeros((1, 64), dtype=torch.int32, device="cuda")
    p = lambda t: C.c_void_p(t.data_ptr())                                   # noqa: E731
    s = C.c_void_p(torch.cuda.current_stream().cuda_stream)
    assert lib.b2t_tracker_step(c.handle, p(d), p(n), None, None, p(out), 256, p(st), 0, s) == EINVAL
    assert lib.b2t_tracker_step_feat(a.handle, p(d), p(n), p(fe), None, None, p(out), 256, p(st), 0, s) == EINVAL
    assert lib.b2t_tracker_set_thetas(c.handle, 1.0, 0.25) == EINVAL
    cfg = L.TrackerConfig(**{k: getattr(c.cfg, k) for k, _ in L.TrackerConfig._fields_})
    cfg.theta_iou = 1.0
    assert lib.b2t_tracker_state_bytes(C.byref(cfg)) == 0
    cfg.theta_iou, cfg.cap, cfg.dmax, cfg.ecap, cfg.n_seq, cfg.feat_dim = 0.5, 1152, 576, 147456, 8, 512     # the C4 configuration
    assert lib.b2t_tracker_state_bytes(C.byref(cfg)) > 0
    torch.cuda.synchronize()


def test_dropin_botsort_with_reid_extractor():
    """The drop-in BoTSORT(use_apperance_model=True) with a seeded ReidExtractor on uint8 frames equals the oracle fed the same
    features, and those come from ONE features_from_frame call per frame on exactly the det_high crops.  The extractor's fp16
    network with batch statistics is not bit-reproducible from call to call (it agrees with itself to ~1e-4), so the features the
    tracker used are recorded and the oracle is fed those; a second call on the same crops must agree with them to 1e-3."""
    from oracle import reid as R
    from b200track.reid import ReidExtractor
    saved = {k: sys.modules.pop(k) for k in list(sys.modules) if k in ("basetrack", "botsort", "matching", "kalman_filter")}
    sys.path.insert(0, os.path.join(PKG, "tracker"))
    try:
        from basetrack import BaseTrack
        from botsort import BoTSORT

        class Opts:
            conf_thresh = 0.2; track_buffer = 30; kalman_format = "botsort"; img_size = 640; iou_thresh = 0.5
            reid_model_path = ""; dhn_path = ""

        class Recording(ReidExtractor):
            def features_from_frame(self, frame, tlbrs):
                out = super().features_from_frame(frame, tlbrs)
                self.calls.append((np.asarray(tlbrs, np.float32).copy(), out.cpu().numpy()))
                return out

        ext = Recording(R.seeded_state_dict(6), bn_mode="batch")
        ext.calls = []
        frames, _, _ = make_reid_stream(21, 12, 40, 32, img=640)
        rng = np.random.default_rng(3)
        BaseTrack._count = 0
        trk = BoTSORT(Opts(), use_GMC=False)
        trk.use_apperance_model = True
        trk.reid_model = ext
        orc = ReidBotsortOracle(use_gmc=False)
        for i, f in enumerate(frames):
            img = rng.integers(0, 256, (640, 640, 3), dtype=np.uint8)
            hi = f[:, 4] >= np.float32(trk.det_thresh)
            ext.calls.clear()
            got = trk.update(f.copy(), img)
            assert len(ext.calls) == 1 and np.array_equal(ext.calls[0][0], f[hi, :4]), "frame %d: one call on the det_high crops" % (i + 1)
            ref_feats = np.zeros((len(f), 512), np.float32)
            ref_feats[hi] = ext.calls[0][1]
            again = ReidExtractor.features_from_frame(ext, img, f[hi, :4]).cpu().numpy()
            np.testing.assert_allclose(again, ext.calls[0][1], rtol=0, atol=1e-3)
            exp = orc.update(f, None, feats=ref_feats)
            assert [t.track_id for t in got] == [e[0] for e in exp], "frame %d" % (i + 1)
            np.testing.assert_allclose(np.array([t.tlwh for t in got]).reshape(-1, 4), np.array([e[1] for e in exp]).reshape(-1, 4),
                                       rtol=1e-9, atol=1e-9)
            ef = orc.last_features()
            for k, t in enumerate(got):
                np.testing.assert_allclose(t.features[-1], ef[k], rtol=0, atol=1e-6)
        assert trk._engine.feat_dim == 512 and int(trk._engine.np_stat[0, L.STAT_NAPP]) >= 0
    finally:
        sys.path.remove(os.path.join(PKG, "tracker"))
        for k in ("basetrack", "botsort", "matching", "kalman_filter"):
            sys.modules.pop(k, None)
        sys.modules.update(saved)


def test_bytetrack_appearance_mode_still_raises():
    saved = {k: sys.modules.pop(k) for k in list(sys.modules) if k in ("basetrack", "bytetrack", "matching", "kalman_filter")}
    sys.path.insert(0, os.path.join(PKG, "tracker"))
    try:
        from bytetrack import ByteTrack

        class Opts:
            conf_thresh = 0.2; track_buffer = 30; kalman_format = "default"; img_size = 640; iou_thresh = 0.5
            reid_model_path = ""; dhn_path = ""

        trk = ByteTrack(Opts())
        trk.use_apperance_model = True
        with pytest.raises(NotImplementedError, match="dense"):
            trk.update(np.zeros((0, 6), np.float32), np.zeros((4, 4, 3), np.uint8))
    finally:
        sys.path.remove(os.path.join(PKG, "tracker"))
        for k in ("basetrack", "bytetrack", "matching", "kalman_filter"):
            sys.modules.pop(k, None)
        sys.modules.update(saved)
