"""Drop-in for the detector side of the reference boundary (SURVEY.md 8b B-det): ``Model`` behaves like the fused,
eval-mode ``models.yolo.Model`` the tracker driver uses (tracker/track.py:82-84,144-145):

    model = attempt_load(weights, map_location=device)      # models/experimental.py
    stride = int(model.stride.max())
    out = model(img.to(device))[0]                          # (B, N, 5 + nc) float32

Two deploy graphs are built: YOLOv7-w6 (cfg/deploy/yolov7-w6.yaml, what the tracker driver loads) and YOLOv7-tiny
(cfg/deploy/yolov7-tiny.yaml, BASELINE.json configs[0]); the forward runs on the wgmma conv kernels through
``b200track.detector.DetectorW6`` / ``b200track.tiny.DetectorTiny``.  Engines are built lazily per (batch, image size)."""
import torch

from . import _b2t_path  # noqa: F401
from b200track.detector import DetectorW6
from b200track import tiny as _tiny
from b200track.w6 import ANCHORS, NC, STRIDES, conv_shapes, fold_reference_state_dict


class Model(torch.nn.Module):
    def __init__(self, cfg="yolov7-w6", ch=3, nc=None, anchors=None, state_dict=None, device="cuda:0"):
        super().__init__()
        self.tiny = "tiny" in str(cfg)
        if "w6" not in str(cfg) and not self.tiny:
            raise NotImplementedError("only the YOLOv7-w6 and YOLOv7-tiny deploy graphs are built for the GPU (SURVEY.md 8a a1)")
        if nc not in (None, NC):
            raise NotImplementedError("nc = %d heads only" % NC)
        self.yaml = {"nc": NC, "anchors": _tiny.ANCHORS if self.tiny else ANCHORS}
        self.nc = NC
        self.names = [str(i) for i in range(NC)]
        self.stride = torch.tensor([float(s) for s in (_tiny.STRIDES if self.tiny else STRIDES)])
        self._device = torch.device(device)
        self._sd = state_dict
        self._engines = {}

    def load_state_dict(self, state_dict, strict=True):
        shapes = conv_shapes(_tiny.tiny_layers(), name_offset=-1) if self.tiny else conv_shapes()
        need = {n + s for n, *_ in shapes for s in (".weight", ".bias")}
        if need - set(state_dict) and self.tiny:
            raise KeyError("YOLOv7-tiny: a fused state dict is expected (model.{i}.conv.weight / .bias, model.77.m.{j}.*): "
                           "Model(cfg).fuse().state_dict() of the reference, or tools/export_state_dict.py")
        if need - set(state_dict):          # unfused (Conv + BN) and / or training-graph (IAuxDetect) naming: fold it
            try:
                state_dict = fold_reference_state_dict(state_dict)
            except KeyError as e:
                if strict:
                    raise KeyError("not a YOLOv7-w6 state dict (deploy, fused, unfused or training graph): %s" % e)
        missing = sorted(need - set(state_dict))
        if missing and strict:
            raise KeyError("missing weights: %s ..." % missing[:3])
        self._sd = {k: v for k, v in state_dict.items() if k in need}
        self._engines.clear()
        return self

    def state_dict(self, *a, **k):
        return dict(self._sd or {})

    def fuse(self):
        return self                       # weights are stored fused (Conv + BN folded, utils/torch_utils.py:181-201)

    def float(self):
        return self

    def half(self):
        return self                       # activations are fp16 on the tensor cores (fp32 accumulation) whatever the caller asks for

    def eval(self):
        return self

    def to(self, device, *a, **k):
        self._device = torch.device(device) if not isinstance(device, torch.dtype) else self._device
        return self

    def _engine(self, batch, size):
        key = (batch, size)
        if key not in self._engines:
            if self._sd is None:
                raise RuntimeError("no weights loaded")
            # graphed: model(img) replays the forward + decode as one CUDA graph; tuned once per (batch, size)
            make = _tiny.DetectorTiny if self.tiny else DetectorW6
            self._engines[key] = make(self._sd, batch=batch, img_size=size, device=self._device, use_graph=True)
        return self._engines[key]

    def forward(self, x, augment=False, profile=False):
        if augment:
            raise NotImplementedError("test-time augmentation is out of scope (SURVEY.md 2.1 row 9)")
        b, c, h, w = x.shape
        st = int(self.stride.max())
        if h % st or w % st:
            raise ValueError("image sides must be multiples of the model stride %d (check_img_size / letterbox(stride) guarantee it, "
                             "tracker/track.py:84, tracker_dataloader.py:100-126); got %d x %d" % (st, h, w))
        eng = self._engine(b, h if h == w else (h, w))       # minimum-rectangle letterboxes (e.g. 768 x 1280, 960 x 1280) get their own engine
        pred = eng.forward(x.to(self._device, torch.float32))
        # fresh tensors, like the reference (the engine's buffers are overwritten by the next call); raw maps in the reference's
        # (B, na, ny, nx, no) layout (models/yolo.py:47-48)
        raw = [r[..., :255].reshape(b, r.shape[1], r.shape[2], 3, NC + 5).permute(0, 3, 1, 2, 4).contiguous() for r in eng.raw]
        return pred.clone(), raw
