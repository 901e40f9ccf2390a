"""TEST INFRASTRUCTURE: builds a ``DetectorW6`` launch plan without a GPU.  ``libb200track.so`` is replaced by a recorder whose
entry points return 0, tensors live on the CPU, and every ``b2t_conv_desc`` the planner would hand to the library is captured
(tests/test_detector_plan.py compares it with a committed golden plan and with the oracle's tensor shapes).  Nothing here
computes anything; the product never imports this module."""
import ctypes as C
from unittest import mock

import torch


class RecorderLib:
    def __init__(self):
        self.calls = []
        self.descs = []
        self.launches = []

    @staticmethod
    def _scalar(a):
        if isinstance(a, (int, float)):
            return a
        if isinstance(a, (C.c_int, C.c_float, C.c_longlong, C.c_double, C.c_size_t)):
            return a.value
        if isinstance(a, C.Array) and a._type_ is C.c_float:
            return [float(v) for v in a]
        return "ptr"

    def __getattr__(self, name):
        def fn(*args):
            self.calls.append(name)
            self.launches.append([name] + [self._scalar(a) for a in args])
            if name == "b2t_conv_plan_create":
                d = args[0]._obj
                self.descs.append({f: getattr(d, f) for f, _ in type(d)._fields_})
            if name == "b2t_conv_plan_flops":
                return 1.0
            if name == "b2t_nms_workspace_bytes":
                return 1 << 20
            if name.endswith("last_error"):
                return b""
            return 0
        return fn


def dry_run_plan(batch, img_size, tiny=False, **kw):
    """Returns (detector, [per-conv dict]) for a plan built on CPU tensors.  Pointers are reported relative to their tensors.
    tiny: plan the YOLOv7-tiny graph (``b200track.tiny.DetectorTiny``) instead of w6."""
    from b200track import _lib as L
    from b200track import detector as D
    from b200track import tiny as T
    from b200track.w6 import seeded_state_dict
    rec = RecorderLib()
    make = (lambda **a: T.DetectorTiny(T.seeded_state_dict(0), **a)) if tiny else (lambda **a: D.DetectorW6(seeded_state_dict(0), **a))
    with mock.patch.object(L, "load", lambda: rec), mock.patch.object(torch.cuda, "is_available", lambda: True):
        det = make(batch=batch, img_size=img_size, device="cpu", use_graph=False, autotune=False, **kw)
    # run every op once against the recorder: the scalar arguments of each C-ABI call become part of the plan
    rec.launches = []

    class _Stream:
        cuda_stream = 0
    with mock.patch.object(torch.cuda, "current_stream", lambda *a, **k: _Stream()):
        det._forward_launches(); det.decode(); det._nms_launch(True); det.nms_from_pred(True)
    det.launch_log = [l for l in rec.launches]
    plans = [p for p in det.keep if hasattr(p, "keep") and isinstance(getattr(p, "keep"), tuple)]
    assert len(plans) == len(rec.descs)
    out = []
    for plan, d in zip(plans, rec.descs):
        x, w, b, y = plan.keep
        e = {k: v for k, v in d.items() if k not in ("x", "w_packed", "bias", "y")}
        e["x_off"] = int(d["x"]) - x.data_ptr()
        e["y_off"] = int(d["y"]) - y.data_ptr()
        e["x_shape"], e["y_shape"], e["w_shape"] = list(x.shape), list(y.shape), list(w.shape)
        e["y_dtype"] = str(y.dtype)
        out.append(e)
    return det, out
