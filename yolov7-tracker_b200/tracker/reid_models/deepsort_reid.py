"""Drop-in for the reference's ``tracker/reid_models/deepsort_reid.py``: ``Extractor(model_path, use_cuda=True)`` with
``__call__(im_crops) -> (n, 512) float32 ndarray`` (reference :109-153), imported by ``basetrack`` / ``botsort`` / ``deepsort`` /
``strongsort`` as ``from reid_models.deepsort_reid import Extractor``.

The network (``Net(reid=True)``, :63-106) runs on the GPU through ``b200track/reid.py``: convolutions on the wgmma kernel, the
rest as element-wise kernels (csrc/b2t_reid.cu).  The reference never switches its network to ``eval()``, so its BatchNorm layers use
the statistics of the crops of each call; ``bn_mode='batch'`` (default) reproduces that, ``'running'`` is eval-mode BatchNorm."""
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import _b2t_path  # noqa: F401,E402
from b200track.reid import ReidExtractor  # noqa: E402


class Extractor(object):
    def __init__(self, model_path, use_cuda=True, bn_mode="batch"):
        if not (use_cuda and torch.cuda.is_available()):
            raise RuntimeError("reid_models.deepsort_reid.Extractor runs on the GPU only (there is no CPU fallback)")
        ckpt = torch.load(model_path, map_location="cpu", weights_only=False)
        state_dict = ckpt["net_dict"] if isinstance(ckpt, dict) and "net_dict" in ckpt else ckpt
        self.net = ReidExtractor(state_dict, device="cuda:%d" % torch.cuda.current_device(), bn_mode=bn_mode)
        self.device = "cuda"
        self.size = (64, 128)

    def __call__(self, im_crops):
        return self.net(im_crops)
