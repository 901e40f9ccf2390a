"""Build container only: runs the UNMODIFIED reference's StrongSORT appearance path (tracker/strongsort.py ``reid_preprocess`` :47-64,
called unbound -- it reads no state -- and ``osnet_x0_25`` of tracker/reid_models/OSNet.py) on seeded crops and seeded weights and
stores what it returns in tests/golden/osnet.npz.

The weights (oracle.osnet.seeded_state_dict(SEED)) reach the network the way StrongSORT loads its checkpoint: saved to a temporary file
with a ``module.`` prefix and an odd-sized classifier, then ``load_model_tools.load_pretrained_weights`` (which strips the prefix and
drops the classifier), then ``eval()``.  Stored: ``pre`` the preprocessed crops (n, 3, 128, 256) float32 at the flat positions
``pre_idx`` (PRE_SAMPLES seeded positions per crop: the whole tensors would be 4.7 MB), ``feat`` the features (n, 512) float32; the crops
are rebuilt by the tests from oracle.reid.seeded_crops(CROP_SEED, N)."""
import contextlib
import importlib
import io
import os
import sys
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)

SEED, CROP_SEED, N, PRE_SAMPLES = 0, 21, 12, 4096


def reference_modules():
    """strongsort, reid_models.OSNet and reid_models.load_model_tools imported from the reference tree (lap / cython_bbox backed by the
    oracle's stand-ins, as oracle/refshim.py does)."""
    import types
    from oracle import iou, lapjv, refshim
    if not hasattr(np, "float"):
        np.float = float
    for name, mod in (("lap", types.SimpleNamespace(lapjv=lapjv.lapjv)), ("cython_bbox", types.SimpleNamespace(bbox_overlaps=iou.bbox_overlaps))):
        m = types.ModuleType(name)
        m.__dict__.update(vars(mod))
        sys.modules.setdefault(name, m)
    for name in ("matplotlib", "matplotlib.pyplot", "seaborn"):
        try:
            importlib.import_module(name)
        except Exception:
            sys.modules[name] = types.ModuleType(name)
    # the reference imports its modules by bare name; the product's same-named drop-ins must neither shadow them nor be shadowed afterwards
    bare = ("reid_models", "strongsort", "basetrack", "matching", "botsort", "kalman_filter")
    ours = lambda k: k in bare or k.startswith("reid_models.")                  # noqa: E731
    saved = {k: sys.modules.pop(k) for k in [k for k in sys.modules if ours(k)]}
    sys.path.insert(0, os.path.join(refshim.REF_ROOT, "tracker"))
    try:
        return (importlib.import_module("strongsort"), importlib.import_module("reid_models.OSNet"),
                importlib.import_module("reid_models.load_model_tools"))
    finally:
        sys.path.pop(0)
        for k in [k for k in sys.modules if ours(k)]:
            sys.modules.pop(k)
        sys.modules.update(saved)


if __name__ == "__main__":
    import torch
    from oracle import osnet as O
    strongsort, osnet_mod, tools = reference_modules()
    crops = O.seeded_crops(CROP_SEED, N)
    pre = torch.stack([strongsort.StrongSORT.reid_preprocess(None, c) for c in crops]).float()
    sd = O.seeded_state_dict(SEED)
    ck = {"module." + k: v for k, v in sd.items() if not k.startswith("classifier")}
    ck["module.classifier.weight"] = torch.randn(1041, 512)
    ck["module.classifier.bias"] = torch.randn(1041)
    model = osnet_mod.osnet_x0_25(num_classes=1, pretrained=False)
    with tempfile.TemporaryDirectory() as d:
        path = os.path.join(d, "osnet_x0_25.pth")
        torch.save(ck, path)
        with contextlib.redirect_stdout(io.StringIO()):
            tools.load_pretrained_weights(model, path)
    model.eval()
    with torch.no_grad():
        feat = model(pre).numpy()
    idx = np.random.default_rng(CROP_SEED).choice(3 * 128 * 256, PRE_SAMPLES, replace=False).astype(np.int64)
    np.savez_compressed(os.path.join(ROOT, "tests", "golden", "osnet.npz"), pre_idx=idx, pre=pre.numpy().reshape(N, -1)[:, idx],
                        feat=feat.astype(np.float32))
    print(pre.shape, feat.shape, float(np.linalg.norm(feat, axis=1).mean()), float((feat == 0).mean()))
