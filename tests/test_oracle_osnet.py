"""not-gpu: oracle/osnet.py (StrongSORT's preprocessing and OSNet x0.25 restated) against tests/golden/osnet.npz, written by the
UNMODIFIED reference (tests/golden/make_golden_osnet.py); the seeded weights are well-conditioned; the drop-in module carries the
reference's parameter names and shapes; and, where the reference tree exists, the oracle against the reference's own network on the real
checkpoint (weights/osnet_x0_25.pth)."""
import os
import sys

import numpy as np
import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "golden"))
from make_golden_osnet import CROP_SEED, N, SEED  # noqa: E402
from oracle import osnet as O  # noqa: E402
from oracle import refshim  # noqa: E402

GOLD = np.load(os.path.join(HERE, "golden", "osnet.npz"))


@pytest.fixture(scope="module")
def pre():
    return O.preprocess(O.seeded_crops(CROP_SEED, N))


def test_preprocess_matches_reference(pre):
    # cv2.resize on float32 and the oracle's float32 taps agree to a few float32 ulps (observed max 9.5e-7 on values below 2.7)
    got = pre.numpy().reshape(N, -1)[:, GOLD["pre_idx"]]
    np.testing.assert_allclose(got, GOLD["pre"], rtol=0, atol=4e-6)


def test_features_match_reference(pre):
    with torch.no_grad():
        f = O.forward(O.seeded_state_dict(SEED), pre).numpy()
    ref = GOLD["feat"]
    # fp32 noise: the same float32 network up to convolution algorithm order (observed max relative L2 ~1e-6)
    rel = np.linalg.norm(f - ref, axis=1) / np.linalg.norm(ref, axis=1)
    assert rel.max() < 1e-4, rel.max()
    assert np.array_equal(f == 0, ref == 0) or np.abs(f - ref).max() < 1e-4


def test_seeded_weights_are_well_conditioned(pre):
    trace = []
    with torch.no_grad():
        f = O.forward(O.seeded_state_dict(SEED), pre, trace)
    norms = f.norm(dim=1)
    zeros = float((f == 0).float().mean())
    assert 5 < float(norms.min()) and float(norms.max()) < 300, norms          # the real checkpoint: 25 on average
    assert 0.15 < zeros < 0.6, zeros                     # the real checkpoint gives ~0.37 on these crops
    gates = torch.cat([torch.cat(g, 1) for _, g in trace], 1)
    assert float(((gates < 0.02) | (gates > 0.98)).float().mean()) < 0.05, "gate sigmoids saturated"
    assert float(gates.std()) > 0.05, "gates all alike: sharing would not be tested"


def test_state_dict_keys_match_checkpoint_layout():
    shapes = O.state_dict_shapes(1041)
    assert len(shapes) == 567
    sd = O.seeded_state_dict(SEED)
    assert [k for k, _ in O.state_dict_shapes(1)] == list(sd)


def test_dropin_module_names_and_shapes():
    sys.path.insert(0, os.path.join(os.path.dirname(HERE), "yolov7-tracker_b200", "tracker"))
    try:
        from reid_models import OSNet as D
    finally:
        sys.path.pop(0)
        for k in [k for k in sys.modules if k == "reid_models" or k.startswith("reid_models.")]:
            sys.modules.pop(k)
    m = D.osnet_x0_25(num_classes=1, pretrained=False)
    assert [(k, tuple(v.shape)) for k, v in m.state_dict().items()] == [(k, tuple(s)) for k, s in O.state_dict_shapes(1)]
    m.load_state_dict(O.seeded_state_dict(SEED))
    with pytest.raises(RuntimeError, match="pretrained=False"):
        D.osnet_x0_25(num_classes=1, pretrained=True)
    for name in ("osnet_x1_0", "osnet_x0_75", "osnet_x0_5", "osnet_ibn_x1_0"):
        with pytest.raises(NotImplementedError):
            getattr(D, name)(num_classes=1, pretrained=False)
    with pytest.raises(RuntimeError, match="eval"):
        m.train()(torch.zeros(1, 3, 128, 256))


@pytest.mark.skipif(not refshim.available() or not os.path.exists(os.path.join(refshim.REF_ROOT, "weights", "osnet_x0_25.pth")),
                    reason="reference tree / checkpoint not present")
def test_oracle_matches_reference_on_real_checkpoint(pre):
    import contextlib
    import io
    from make_golden_osnet import reference_modules
    _, osnet_mod, tools = reference_modules()
    model = osnet_mod.osnet_x0_25(num_classes=1, pretrained=False)
    path = os.path.join(refshim.REF_ROOT, "weights", "osnet_x0_25.pth")
    with contextlib.redirect_stdout(io.StringIO()):
        tools.load_pretrained_weights(model, path)
    model.eval()
    with torch.no_grad():
        ref = model(pre)
        f = O.forward(model.state_dict(), pre)
    rel = (f - ref).norm(dim=1) / ref.norm(dim=1)
    assert float(rel.max()) < 1e-4, rel
