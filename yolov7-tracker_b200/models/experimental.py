"""``attempt_load`` (reference models/experimental.py:83-106) for the H100 detector.

The reference un-pickles a whole ``nn.Module`` from the checkpoint (key 'ema' or 'model').  Pickled reference modules
cannot be loaded without the reference's own class definitions, so this loader accepts
  * a ``.pt`` file holding a *state dict* of the fused reference model (``model.fuse().state_dict()``), or a dict
    with that state dict under 'model' / 'ema' / 'state_dict';
  * the string ``'seeded:<seed>[:<img_size>]'`` -- the LSUV-calibrated random weights the benches use (the reference
    ships no detector checkpoint, SURVEY.md 2.1 row 23).
A pickled reference checkpoint (``ckpt['ema' or 'model']`` is an ``nn.Module``, models/experimental.py:88-89) is converted once with
``tools/export_state_dict.py`` run next to the reference's code; ``attempt_load`` names that tool when it meets such a file."""
import torch

from . import _b2t_path  # noqa: F401
from .yolo import Model


def attempt_load(weights, map_location=None):
    device = map_location if map_location is not None else "cuda:0"
    if isinstance(weights, (list, tuple)):
        if len(weights) != 1:
            raise NotImplementedError("model ensembles are out of scope")
        weights = weights[0]
    if isinstance(weights, str) and weights.startswith("seeded:"):
        from b200track.w6 import calibrated_state_dict
        parts = weights.split(":")
        sd = calibrated_state_dict(int(parts[1]), int(parts[2]) if len(parts) > 2 else 1280, device)
    else:
        try:
            ckpt = torch.load(weights, map_location="cpu", weights_only=True)
        except Exception as e:                                # pickled nn.Module: needs the reference's own classes to un-pickle
            raise RuntimeError("%s is not a plain state dict (%s: %s).  The reference's checkpoints pickle the whole nn.Module; convert once with\n"
                               "    python tools/export_state_dict.py --reference <Yolov7-tracker checkout> --weights %s --out w6_state.pt\n"
                               "and load w6_state.pt (INTEGRATION.md section 2)." % (weights, type(e).__name__, str(e).split("\n")[0][:120], weights)) from None
        sd = ckpt
        for key in ("ema", "model", "state_dict"):
            if isinstance(ckpt, dict) and key in ckpt and isinstance(ckpt[key], dict):
                sd = ckpt[key]
                break
    # which graph?  The Detect head sits at module 77 in YOLOv7-tiny (cfg/deploy/yolov7-tiny.yaml:111), at 118 / 122 in w6
    cfg = "yolov7-tiny" if any(k.startswith("model.77.m.") for k in sd) and not any(k.startswith("model.118.") for k in sd) else "yolov7-w6"
    return Model(cfg, device=device).load_state_dict({k: v.float() for k, v in sd.items()})
