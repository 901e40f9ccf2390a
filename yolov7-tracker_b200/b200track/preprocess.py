"""Frame pre-processing on the GPU (csrc/b2t_preproc.cu): what ``TrackerLoader.__getitem__`` does per frame in the reference
(tracker/tracker_dataloader.py:64-96, 'v5' / 'v7' branch) -- letterbox resize + 114 border, BGR -> RGB, CHW, float / 255 --
starting from the uint8 BGR frame as ``cv2.imread`` returns it.  The frame crosses PCIe as uint8 (3 bytes per pixel instead
of the 12 of the float tensor the reference uploads) and the result is produced directly in device memory.
"""
import ctypes as C

import numpy as np
import torch

from . import _lib as L


def letterbox_geometry(shape_hw, new_shape=(1280, 1280), stride=32, auto=True, scaleup=True):
    """Host arithmetic of ``_letterbox`` (tracker_dataloader.py:100-126): the resized size, the borders and the ratio.
    Python's round() and numpy's mod are what the reference uses; kept operation for operation."""
    h, w = int(shape_hw[0]), int(shape_hw[1])
    if isinstance(new_shape, int):
        new_shape = (new_shape, new_shape)
    r = min(new_shape[0] / h, new_shape[1] / w)
    if not scaleup:
        r = min(r, 1.0)
    unpad_w, unpad_h = int(round(w * r)), int(round(h * r))
    dw, dh = new_shape[1] - unpad_w, new_shape[0] - unpad_h
    if auto:                                            # minimum rectangle: pad only up to the next stride multiple
        dw, dh = np.mod(dw, stride), np.mod(dh, stride)
    dw, dh = dw / 2, dh / 2
    top, bottom = int(round(dh - 0.1)), int(round(dh + 0.1))
    left, right = int(round(dw - 0.1)), int(round(dw + 0.1))
    return {"unpad_w": unpad_w, "unpad_h": unpad_h, "top": top, "bottom": bottom, "left": left, "right": right,
            "out_h": unpad_h + top + bottom, "out_w": unpad_w + left + right, "ratio": (r, r), "pad": (float(dw), float(dh))}


def scale_coords_geometry(canvas_hw, src_hw):
    """(gain, pad_w, pad_h) of ``scale_coords(img1_shape, coords, img0_shape, ratio_pad=None)`` (utils/general.py:319-332), the call
    tracker/track.py:240 makes to map NMS rows from the (H, W) canvas back to the (h, w) source frame.  Recomputed from the two
    shapes as the reference does, not taken from the letterbox: for 721 x 1283 -> 768 x 1280 it gives pad_h 24.3429, where the
    letterbox placed the image at 24.5.  Same-size frames give (1.0, 0.0, 0.0)."""
    gain = min(canvas_hw[0] / src_hw[0], canvas_hw[1] / src_hw[1])
    return gain, (canvas_hw[1] - src_hw[1] * gain) / 2, (canvas_hw[0] - src_hw[0] * gain) / 2


def launch_letterbox(lib, src_ptr, batch, h, w, pitch, geo, out_ptr, stream_ptr, pad_value=114):
    """One call of the C ABI entry point on raw pointers (also how tests/hostsim drives the simulator build)."""
    rc = lib.b2t_letterbox(C.c_void_p(src_ptr), batch, h, w, pitch, geo["unpad_w"], geo["unpad_h"], geo["top"], geo["left"], geo["out_h"], geo["out_w"],
                           pad_value, C.c_void_p(out_ptr), stream_ptr)
    if rc != 0:
        raise L.B2TError("b2t_letterbox: %s" % (lib.b2t_detect_last_error() or b"").decode())


def launch_letterbox_reorg(lib, src_ptr, batch, h, w, pitch, geo, out_ptr, row_pixels, x0, stream_ptr, pad_value=114, act_dtype=L.ACT_F16):
    """b2t_letterbox_reorg on raw pointers: the letterboxed canvas straight into the detector's padded ReOrg / NHWC 16-bit buffer
    (``DetectorW6.place[0]``: rows of ``stem_row`` pixels, image at pixel 1) -- the uint8 ingest path of ``TrackingPipeline``."""
    rc = lib.b2t_letterbox_reorg(C.c_void_p(src_ptr), batch, h, w, pitch, geo["unpad_w"], geo["unpad_h"], geo["top"], geo["left"], geo["out_h"],
                                 geo["out_w"], pad_value, C.c_void_p(out_ptr), row_pixels, x0, act_dtype, stream_ptr)
    if rc != 0:
        raise L.B2TError("b2t_letterbox_reorg: %s" % (lib.b2t_detect_last_error() or b"").decode())


class Letterbox:
    """``img, geo = Letterbox(new_shape, stride)(frames)``: frames = uint8 BGR ``(H, W, 3)`` or ``(B, H, W, 3)``, numpy (copied from
    pinned memory) or a CUDA tensor; img = float32 ``(B, 3, H', W')`` in [0, 1] on the device -- the tensor the reference hands
    to the model after ``.to(device)`` (tracker/track.py:143-145)."""

    def __init__(self, new_shape=1280, stride=32, device="cuda:0", auto=True):
        if not torch.cuda.is_available():
            raise L.B2TError("Letterbox needs a CUDA device: there is no CPU fallback")
        self.lib = L.load()
        self.new_shape = (new_shape, new_shape) if isinstance(new_shape, int) else tuple(new_shape)
        self.stride, self.auto, self.dev = stride, auto, torch.device(device)
        self._pinned = self._dev_u8 = None

    def __call__(self, frames):
        if isinstance(frames, np.ndarray):
            a = frames if frames.ndim == 4 else frames[None]
            if a.dtype != np.uint8 or a.shape[-1] != 3:
                raise ValueError("frames must be uint8 BGR (H, W, 3)")
            if self._pinned is None or tuple(self._pinned.shape) != a.shape:
                self._pinned = torch.empty(a.shape, dtype=torch.uint8).pin_memory()
                self._dev_u8 = torch.empty(a.shape, dtype=torch.uint8, device=self.dev)
            self._pinned.numpy()[...] = a
            self._dev_u8.copy_(self._pinned, non_blocking=True)
            u8 = self._dev_u8
        else:
            u8 = frames if frames.dim() == 4 else frames[None]
            if u8.dtype != torch.uint8 or not u8.is_cuda or u8.shape[-1] != 3:
                raise ValueError("frames must be a uint8 BGR CUDA tensor (H, W, 3)")
            u8 = u8.contiguous()
        b, h, w, _ = u8.shape
        geo = letterbox_geometry((h, w), self.new_shape, self.stride, self.auto)
        out = torch.empty((b, 3, geo["out_h"], geo["out_w"]), dtype=torch.float32, device=self.dev)
        with torch.cuda.device(self.dev):
            launch_letterbox(self.lib, u8.data_ptr(), b, h, w, 3 * w, geo, out.data_ptr(), C.c_void_p(torch.cuda.current_stream(self.dev).cuda_stream))
        return out, geo
