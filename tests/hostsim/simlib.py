"""TEST INFRASTRUCTURE: drives libb2t_hostsim.so (kernels compiled for the fiber simulator) with
NumPy arrays standing in for device memory.  Used only by the `not gpu` tests to check kernel
LOGIC in the GPU-less container; GPU results are checked by the `-m gpu` tests."""
import ctypes as C
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import build_sim  # noqa: E402

from b200track import _lib as L  # noqa: E402  (only the ctypes declarations are shared)

_sim = None


def sim():
    global _sim
    if _sim is None:
        _sim = L.declare(C.CDLL(build_sim.build()), names=L.TRACKER_SYMBOLS + L.NMS_SYMBOLS + L.REID_SYMBOLS)   # the TUs build_sim compiles
    return _sim


def ptr(a):
    return None if a is None else a.ctypes.data_as(C.c_void_p)


def npdt(dtype):
    return np.float64 if dtype == L.F64 else np.float32


class SimTracker:
    def __init__(self, kind="bytetrack", dtype=L.F64, n_seq=1, cap=512, dmax=512, ecap=8192, kalman_format=None,
                 conf_thresh=0.2, iou_thresh=0.5, track_buffer=30, frame_rate=30, use_gmc=True):
        lib = sim()
        if kalman_format is None:
            kalman_format = "botsort" if kind == "botsort" else "default"
        self.cfg = L.TrackerConfig(kind=L.KIND_BY_NAME[kind], dtype=dtype, fmt=L.FMT_BY_NAME[kalman_format], n_seq=n_seq,
                                   cap=cap, dmax=dmax, ecap=ecap, use_gmc=int(use_gmc), track_buffer=track_buffer,
                                   conf_thresh=conf_thresh, iou_thresh=iou_thresh, frame_rate=frame_rate)
        nbytes = lib.b2t_tracker_state_bytes(C.byref(self.cfg))
        assert nbytes > 0, lib.b2t_last_error()
        self.mem = np.zeros(nbytes + 256, dtype=np.uint8)
        off = (-self.mem.ctypes.data) % 256
        self.h = C.c_void_p()
        L.check(lib, lib.b2t_tracker_create(C.byref(self.cfg), C.c_void_p(self.mem.ctypes.data + off), None, C.byref(self.h)))
        self.S, self.cap, self.dmax = n_seq, cap, dmax
        self.out = np.zeros((n_seq, cap, L.OUT_COLS), np.float64)
        self.stat = np.zeros((n_seq, L.STAT_WORDS), np.int32)

    def step(self, dets_list, warps=None, id_base=None, predict_only=False):
        """dets_list: per sequence an (n,6) float32 array."""
        lib = sim()
        d = np.zeros((self.S, self.dmax, 6), np.float32)
        cnt = np.zeros(self.S, np.int32)
        for s, a in enumerate(dets_list):
            a = np.asarray(a, np.float32).reshape(-1, 6)
            d[s, :len(a)] = a
            cnt[s] = len(a)
        w = None if warps is None else np.ascontiguousarray(np.asarray(warps, np.float64).reshape(self.S, 6))
        ib = None if id_base is None else np.ascontiguousarray(np.asarray(id_base, np.int32))
        L.check(lib, lib.b2t_tracker_step_host(self.h, ptr(d), ptr(cnt), ptr(w), ptr(ib), ptr(self.out), self.cap,
                                               ptr(self.stat), int(predict_only), None))
        res = []
        for s in range(self.S):
            n = self.stat[s, L.STAT_NOUT]
            res.append(self.out[s, :n].copy())
        return res
