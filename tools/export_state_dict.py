"""One-time converter for the reference's pickled checkpoints (run it where the reference's code lives).

The reference saves / loads whole ``nn.Module`` objects: ``attempt_load`` does ``ckpt = torch.load(w); model = ckpt['ema' if
ckpt.get('ema') else 'model'].float().fuse().eval()`` (models/experimental.py:83-106).  Un-pickling needs the reference's own
``models`` / ``utils`` packages on ``sys.path``; the GPU detector only needs the tensors.  This script does the reference's own
load + ``.float()`` and writes ``model.state_dict()`` -- deploy, unfused (Conv + BN) or training-graph (IAuxDetect) naming, all of
which ``b200track.w6.fold_reference_state_dict`` folds on load:

    python tools/export_state_dict.py --reference /path/to/Yolov7-tracker --weights yolov7-w6.pt --out w6_state.pt
    # then, in tracker/track.py's place:  attempt_load('w6_state.pt', map_location=device)
"""
import argparse
import sys

import torch


def export(reference, weights, out):
    sys.path.insert(0, reference)                      # the checkpoint's pickled classes are models.yolo.Model, models.common.* ...
    ckpt = torch.load(weights, map_location="cpu", weights_only=False)
    model = ckpt["ema" if isinstance(ckpt, dict) and ckpt.get("ema") is not None else "model"] if isinstance(ckpt, dict) else ckpt
    sd = {k: v.float() for k, v in model.float().state_dict().items() if torch.is_tensor(v) and v.is_floating_point()}
    torch.save(sd, out)
    return len(sd)


if __name__ == "__main__":
    ap = argparse.ArgumentParser()
    ap.add_argument("--reference", required=True, help="checkout of the reference repository (its models/ and utils/ packages)")
    ap.add_argument("--weights", required=True)
    ap.add_argument("--out", required=True)
    a = ap.parse_args()
    print("wrote %d tensors to %s" % (export(a.reference, a.weights, a.out), a.out))
