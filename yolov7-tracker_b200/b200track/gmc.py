"""Camera-motion estimation on the GPU: host side of csrc/b2t_gmc.cu (SURVEY.md section 8f row 1) and csrc/b2t_ecc.cu.

``GmcEstimator`` is what ``tracker/botsort.py:GMC(method='orb')`` runs on: the reference's ``GMC.applyFeaures``
(tracker/botsort.py:111-235 -- FAST + ORB key points outside the detection boxes, 2-NN Hamming matching against the previous
frame, ratio / spatial / 2.5 sigma filters, RANSAC partial affine) as eleven kernel launches per call for any number of
sequences, state (previous key points and descriptors) in a caller-owned device workspace.  ``EccEstimator`` is what
``GMC(method='ecc')`` runs on (the reference's ``GMC.applyEcc``, tracker/botsort.py:78-109).  PyTorch only owns the memory.
"""
import ctypes as C

import numpy as np

from . import _lib as L


def _check(lib, rc):
    if rc != 0:
        raise L.B2TError("libb200track error %d: %s" % (rc, (lib.b2t_detect_last_error() or b"").decode()))


def workspace_layout(lib, n_seq, height, width, downscale, max_kp):
    out = (C.c_size_t * 10)()
    _check(lib, lib.b2t_gmc_workspace_layout(n_seq, height, width, downscale, max_kp, out, 10))
    keys = ("stride", "state", "gray", "blur", "score", "kp", "desc", "h", "w", "pts")
    return dict(zip(keys, [int(v) for v in out]))


def launch_estimate(lib, frames_ptr, n_seq, height, width, pitch, downscale, dets_ptr, counts_ptr, dmax, det_thresh, ws_ptr, max_kp,
                    warps_ptr, stat_ptr, stream):
    _check(lib, lib.b2t_gmc_estimate(frames_ptr, n_seq, height, width, pitch, downscale, dets_ptr, counts_ptr, dmax, float(det_thresh),
                                     ws_ptr, max_kp, warps_ptr, stat_ptr, stream))


def unpack_keypoints(ws_bytes, layout, seq, buf, n, max_kp):
    """(xs, ys, descriptors (n, 32) uint8) of key-point buffer `buf` of sequence `seq` from a host copy of the workspace (tests)."""
    base = seq * layout["stride"]
    kp = np.frombuffer(ws_bytes, np.uint32, max_kp, base + layout["kp"] + buf * max_kp * 4)[:n]
    desc = np.frombuffer(ws_bytes, np.uint8, max_kp * 32, base + layout["desc"] + buf * max_kp * 32).reshape(max_kp, 32)[:n]
    return (kp & 0xffff).astype(np.int64), (kp >> 16).astype(np.int64), desc


class GmcEstimator:
    """One estimator for ``n_seq`` sequences of (height, width) BGR frames.  ``estimate`` enqueues on the current stream and
    returns device tensors (no synchronisation): warps (n_seq, 2, 3) float64 -- what ``TrackEngine.step_device(warps=...)``
    takes -- and the stat words."""

    def __init__(self, n_seq, height, width, downscale=2, max_kp=8192, device="cuda:0"):
        import torch
        self.torch = torch
        if not torch.cuda.is_available():
            raise L.B2TError("GmcEstimator needs a CUDA device (there is no CPU fallback)")
        self.lib = L.load()
        self.S, self.h, self.w, self.ds, self.max_kp = int(n_seq), int(height), int(width), max(1, int(downscale)), int(max_kp)
        self.dev = torch.device(device)
        nbytes = self.lib.b2t_gmc_workspace_bytes(self.S, self.h, self.w, self.ds, self.max_kp)
        if nbytes == 0:
            raise L.B2TError("b2t_gmc_workspace_bytes: unsupported geometry %dx%d / %d (at least 64 px per side after down-scaling)" % (self.h, self.w, self.ds))
        self.layout = workspace_layout(self.lib, self.S, self.h, self.w, self.ds, self.max_kp)
        self.ws = torch.zeros(nbytes, dtype=torch.uint8, device=self.dev)
        self.warps = torch.zeros((self.S, 2, 3), dtype=torch.float64, device=self.dev)
        self.stat = torch.zeros((self.S, L.GMC_STAT_WORDS), dtype=torch.int32, device=self.dev)
        self.launches_per_call = 11

    def reset(self):
        with self.torch.cuda.device(self.dev):
            _check(self.lib, self.lib.b2t_gmc_reset(self.ws.data_ptr(), self.S, self.h, self.w, self.ds, self.max_kp,
                                                    self.torch.cuda.current_stream().cuda_stream))

    def estimate(self, frames, dets=None, det_counts=None, det_thresh=float("-inf")):
        """frames: (n_seq, height, width, 3) uint8 BGR device tensor; dets: (n_seq, dmax, 6) float32 device tensor with
        det_counts (n_seq,) int32 (the NMS output buffers) or None.  Boxes of detections with score >= det_thresh are masked out."""
        t = self.torch
        if frames.dtype != t.uint8 or tuple(frames.shape) != (self.S, self.h, self.w, 3) or not frames.is_contiguous() or frames.device != self.dev:
            raise L.B2TError("frames must be a contiguous uint8 (%d, %d, %d, 3) tensor on %s" % (self.S, self.h, self.w, self.dev))
        dmax, dp, cp = 0, None, None
        if dets is not None:
            if dets.dtype != t.float32 or dets.dim() != 3 or dets.shape[0] != self.S or dets.shape[2] != 6 or not dets.is_contiguous() or dets.device != self.dev:
                raise L.B2TError("dets must be a contiguous float32 (n_seq, dmax, 6) tensor on the estimator's device")
            dmax, dp = int(dets.shape[1]), dets.data_ptr()
            if det_counts is not None:
                if det_counts.dtype != t.int32 or tuple(det_counts.shape) != (self.S,) or det_counts.device != self.dev:
                    raise L.B2TError("det_counts must be an int32 (n_seq,) tensor on the estimator's device")
                cp = det_counts.data_ptr()
        with t.cuda.device(self.dev):
            launch_estimate(self.lib, frames.data_ptr(), self.S, self.h, self.w, 3 * self.w, self.ds, dp, cp, dmax, det_thresh,
                            self.ws.data_ptr(), self.max_kp, self.warps.data_ptr(), self.stat.data_ptr(), t.cuda.current_stream().cuda_stream)
        return self.warps, self.stat

    def prepare(self, frames, slot):
        """First half of ``estimate`` (gray image, FAST scores, smoothed image into plane set ``slot``): needs only the frames, so a
        pipeline can run it while the frame buffer is still valid (b200track/pipeline.py)."""
        t = self.torch
        if frames.dtype != t.uint8 or tuple(frames.shape) != (self.S, self.h, self.w, 3) or not frames.is_contiguous() or frames.device != self.dev:
            raise L.B2TError("frames must be a contiguous uint8 (%d, %d, %d, 3) tensor on %s" % (self.S, self.h, self.w, self.dev))
        with t.cuda.device(self.dev):
            _check(self.lib, self.lib.b2t_gmc_prepare(frames.data_ptr(), self.S, self.h, self.w, 3 * self.w, self.ds, self.ws.data_ptr(), self.max_kp,
                                                      int(slot), t.cuda.current_stream().cuda_stream))

    def estimate_prepared(self, slot, dets=None, det_counts=None, det_thresh=float("-inf")):
        """Second half: key points outside the detection boxes, descriptors, matching, filters, RANSAC.  Call in frame order."""
        t = self.torch
        dmax = 0 if dets is None else int(dets.shape[1])
        with t.cuda.device(self.dev):
            _check(self.lib, self.lib.b2t_gmc_estimate_prepared(self.S, self.h, self.w, self.ds, None if dets is None else dets.data_ptr(),
                                                                None if det_counts is None else det_counts.data_ptr(), dmax, float(det_thresh),
                                                                self.ws.data_ptr(), self.max_kp, int(slot), self.warps.data_ptr(), self.stat.data_ptr(),
                                                                t.cuda.current_stream().cuda_stream))
        return self.warps, self.stat

    def keypoints(self, seq, which="current"):
        """Host copy of a key-point buffer after ``estimate`` (tests / tools; synchronises)."""
        ws = self.ws.cpu().numpy().tobytes()
        state = np.frombuffer(ws, np.int32, 16, seq * self.layout["stride"] + self.layout["state"])
        buf = (int(state[0]) - 1) & 1                   # estimate() already advanced the frame counter
        if which != "current":
            buf ^= 1
        return unpack_keypoints(ws, self.layout, seq, buf, int(state[1 + buf]), self.max_kp)


def ecc_workspace_layout(lib, n_seq, height, width, downscale):
    out = (C.c_size_t * 6)()
    _check(lib, lib.b2t_ecc_workspace_layout(n_seq, height, width, downscale, out, 6))
    return dict(zip(("stride", "state", "template", "current", "h", "w"), [int(v) for v in out]))


def launch_ecc(lib, frames_ptr, n_seq, height, width, pitch, downscale, max_iter, eps, ws_ptr, warps_ptr, stat_ptr, stream):
    _check(lib, lib.b2t_ecc_estimate(frames_ptr, n_seq, height, width, pitch, downscale, int(max_iter), float(eps), ws_ptr, warps_ptr,
                                     stat_ptr, stream))


def ecc_rho(stat):
    """The final rho of each sequence from the stat words of ``EccEstimator.estimate`` (host int32 array (n_seq, 8))."""
    s = np.ascontiguousarray(np.asarray(stat, np.int32)[:, 1:3])
    return s.view(np.float64)[:, 0]


class EccEstimator:
    """ECC camera-motion estimation (csrc/b2t_ecc.cu) for ``n_seq`` sequences of (height, width) BGR frames: what
    ``tracker/botsort.py:GMC(method='ecc')`` runs on -- the reference's ``GMC.applyEcc`` (tracker/botsort.py:78-109).  Each
    sequence's first frame after construction or ``reset()`` becomes its template and is never replaced (the reference's
    behaviour, quirk q17); later frames are aligned to it with findTransformECC's Euclidean Gauss-Newton loop, all iterations in
    one launch of one thread-block cluster per sequence.  ``estimate`` enqueues on the current stream and returns device tensors
    (no synchronisation): warps (n_seq, 2, 3) float64 holding float32 values, in down-scaled pixels as the reference returns them,
    and the stat words (iterations, rho as two words -- ``ecc_rho`` --, flags ``_lib.ECC_*`` in word 5, frame index in word 7)."""

    def __init__(self, n_seq, height, width, downscale=2, max_iter=100, eps=1e-5, device="cuda:0"):
        import torch
        self.torch = torch
        if not torch.cuda.is_available():
            raise L.B2TError("EccEstimator needs a CUDA device (there is no CPU fallback)")
        self.lib = L.load()
        self.S, self.h, self.w, self.ds = int(n_seq), int(height), int(width), max(1, int(downscale))
        self.max_iter, self.eps = int(max_iter), float(eps)
        if self.max_iter < 1 or not self.eps >= 0.0:
            raise L.B2TError("EccEstimator: max_iter must be >= 1 and eps >= 0")
        self.dev = torch.device(device)
        nbytes = self.lib.b2t_ecc_workspace_bytes(self.S, self.h, self.w, self.ds)
        if nbytes == 0:
            raise L.B2TError("b2t_ecc_workspace_bytes: unsupported geometry %dx%d / %d (at least 8 px per side after down-scaling)" % (self.h, self.w, self.ds))
        self.layout = ecc_workspace_layout(self.lib, self.S, self.h, self.w, self.ds)
        self.ws = torch.zeros(nbytes, dtype=torch.uint8, device=self.dev)
        self.warps = torch.zeros((self.S, 2, 3), dtype=torch.float64, device=self.dev)
        self.stat = torch.zeros((self.S, L.GMC_STAT_WORDS), dtype=torch.int32, device=self.dev)
        self.launches_per_call = 2

    def reset(self):
        """Forget the templates: the next frame of every sequence becomes its new template."""
        with self.torch.cuda.device(self.dev):
            _check(self.lib, self.lib.b2t_ecc_reset(self.ws.data_ptr(), self.S, self.h, self.w, self.ds, self.torch.cuda.current_stream().cuda_stream))

    def estimate(self, frames):
        """frames: (n_seq, height, width, 3) uint8 BGR device tensor."""
        t = self.torch
        if frames.dtype != t.uint8 or tuple(frames.shape) != (self.S, self.h, self.w, 3) or not frames.is_contiguous() or frames.device != self.dev:
            raise L.B2TError("frames must be a contiguous uint8 (%d, %d, %d, 3) tensor on %s" % (self.S, self.h, self.w, self.dev))
        with t.cuda.device(self.dev):
            launch_ecc(self.lib, frames.data_ptr(), self.S, self.h, self.w, 3 * self.w, self.ds, self.max_iter, self.eps, self.ws.data_ptr(),
                       self.warps.data_ptr(), self.stat.data_ptr(), t.cuda.current_stream().cuda_stream)
        return self.warps, self.stat

    def plane(self, seq, which="template"):
        """Host copy of a sequence's prepared plane, 'template' or 'current' (tests / tools; synchronises)."""
        o = seq * self.layout["stride"] + self.layout[which]
        n = self.layout["h"] * self.layout["w"]
        return self.ws[o:o + n].cpu().numpy().reshape(self.layout["h"], self.layout["w"])
