"""-m gpu: the ReID extractor of the appearance branch (SURVEY.md 8f row 3) on an H100 -- wgmma convolutions + the element-wise
kernels of csrc/b2t_reid.cu -- against oracle/reid.py (pinned against the reference's own Net / Extractor and its checkpoint by
tests/test_oracle_reid.py).  fp16 activations: features are compared by cosine similarity and absolute difference."""
import os
import sys

import numpy as np
import pytest

pytestmark = pytest.mark.gpu
torch = pytest.importorskip("torch")

from b200track.reid import ReidExtractor  # noqa: E402
from oracle import reid as R  # noqa: E402


@pytest.mark.parametrize("bn_mode", ["batch", "running"])
def test_extractor_features_vs_oracle(bn_mode):
    sd = R.seeded_state_dict(3)
    crops = R.seeded_crops(21, 11)
    ext = ReidExtractor(sd, bn_mode=bn_mode)
    got = ext(crops)
    assert got.shape == (11, 512) and got.dtype == np.float32
    with torch.no_grad():
        exp = R.forward(sd, R.preprocess(crops), batch_stats=bn_mode == "batch").numpy()
    cos = (got * exp).sum(1)
    print("reid %s: min cosine %.6f, max |d| %.2e" % (bn_mode, float(cos.min()), float(np.abs(got - exp).max())))
    assert np.allclose(np.linalg.norm(got, axis=1), 1.0, atol=1e-4)
    assert cos.min() > 0.9999 and np.abs(got - exp).max() < 2e-3
    # the pre-processing stage on its own: crop -> float / 255 -> bilinear 64 x 128 -> Normalize, fp16-rounded
    x = ext.last_net["x"][:11, :, :, :3].float().cpu().permute(0, 3, 1, 2)
    assert float((x - R.preprocess(crops)).abs().max()) < 3e-3
    assert float(ext.last_net["x"][:, :, :, 3:].abs().max()) == 0.0


def test_features_from_frame_and_cosine_distance():
    """BoTSORT.get_feature's form (crops = windows of the frame, botsort.py:291-311) and the distance matrix of
    matching.embedding_distance (matching.py:84-103) on the wgmma conv kernel."""
    from b200track.gemm import CosineGemm
    from b200track.synth import textured_frame
    sd = R.seeded_state_dict(4)
    frame = textured_frame(77, 480, 640, n_rect=300)
    rng = np.random.default_rng(2)
    x1 = rng.uniform(0, 500, 40); y1 = rng.uniform(0, 300, 40)
    tlbr = np.stack([x1, y1, x1 + rng.uniform(16, 120, 40), y1 + rng.uniform(30, 170, 40)], 1)
    ext = ReidExtractor(sd, bn_mode="batch")
    f = ext.features_from_frame(frame, tlbr)
    t = tlbr.astype(np.int64)
    crops = [frame[a[1]:a[3], a[0]:a[2]] for a in t]
    with torch.no_grad():
        exp = R.forward(sd, R.preprocess(crops), batch_stats=True)
    cos = (f.cpu() * exp).sum(1)
    assert float(cos.min()) > 0.9999
    d = 1.0 - CosineGemm().cosine_similarity(f[:25], f[25:]).cpu().double().numpy()
    fe = f.cpu().double().numpy()
    ref = 1.0 - fe[:25] @ fe[25:].T
    assert np.abs(d - ref).max() < 5e-6


def test_dropin_extractor_module(tmp_path):
    sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "yolov7-tracker_b200", "tracker"))
    try:
        from reid_models.deepsort_reid import Extractor
    finally:
        sys.path.pop(0)
    sd = R.seeded_state_dict(5)
    path = str(tmp_path / "ckpt.t7")
    torch.save({"net_dict": sd, "acc": 0.0, "epoch": 0}, path)              # the layout of the reference's weights/ckpt.t7
    ext = Extractor(path, use_cuda=True)
    crops = R.seeded_crops(8, 3)
    got = ext(crops)
    with torch.no_grad():
        exp = R.forward(sd, R.preprocess(crops), batch_stats=True).numpy()
    assert got.shape == (3, 512) and float((got * exp).sum(1).min()) > 0.9999
    assert ext([]).shape == (0, 512)
