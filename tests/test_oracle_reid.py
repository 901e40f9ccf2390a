"""Pins oracle/reid.py (restatement of tracker/reid_models/deepsort_reid.py) against the UNMODIFIED reference: the committed golden
outputs of the reference's preprocessing and Net on seeded weights (tests/golden/refchecks.npz).  CPU tier."""
import os
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "yolov7-tracker_b200")):
    if p not in sys.path:
        sys.path.insert(0, p)
from oracle import reid as R  # noqa: E402

REFCHECKS = os.path.join(ROOT, "tests", "golden", "refchecks.npz")


def test_restatement_equals_reference_net_and_preprocess():
    """The restated preprocessing against the reference Extractor's (a seeded sample of the batch) and the restated network
    against the reference's own Net on the seeded weights the GPU tier uses, in eval mode and in train mode (batch statistics:
    the reference never switches its extractor to eval()) -- outputs stored in tests/golden/refchecks.npz.  Narrower than a live run
    of the reference: its own checkpoint (46 MB) and its running-buffer update (a train-mode call followed by an eval-mode call with
    the updated buffers) are not covered."""
    g = np.load(REFCHECKS)
    crops = R.seeded_crops(9, 5)
    x = R.preprocess(crops)
    assert tuple(x.shape) == tuple(g["reid_x_shape"])
    assert float(np.abs(x.numpy().reshape(-1)[g["reid_x_index"]] - g["reid_x"]).max()) < 2e-6          # cv2.resize on float data, restated
    seeded = R.seeded_state_dict(3)
    with torch.no_grad():
        assert float(np.abs(R.forward(seeded, x, batch_stats=False).numpy() - g["reid_eval"]).max()) < 2e-5
        assert float(np.abs(R.forward(seeded, x, batch_stats=True).numpy() - g["reid_train"]).max()) < 2e-5


def test_seeded_network_is_well_conditioned():
    """The seeded stand-in weights give distinct, unit-norm features (the GPU parity test is meaningful on them)."""
    with torch.no_grad():
        f = R.forward(R.seeded_state_dict(3), R.preprocess(R.seeded_crops(1, 6)), batch_stats=True)
    assert torch.allclose(f.norm(dim=1), torch.ones(6), atol=1e-5)
    cos = (f @ f.T).numpy()
    assert np.all(cos[~np.eye(6, dtype=bool)] < 0.999)
