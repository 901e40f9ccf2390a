"""Drop-in for the reference's ``tracker/botsort.py``: ``BoTSORT(opts, frame_rate=30, gamma=0.02,
use_GMC=True)``, ``multi_gmc`` and ``GMC``.

``BoTSORT.update`` (reference :313-493) runs as one fused kernel per frame (kind = botsort): Kalman
predict, ``multi_gmc`` of the pool and of the unconfirmed tracks (:380-382), three IoU associations,
births from ALL first-stage leftovers (q3), list algebra.  ``multi_gmc`` (:250-269) is also
available on its own for lists of STrack (b2t_gmc_apply).

Camera-motion ESTIMATION (``GMC.apply``, method 'orb', reference :111-235 -- SURVEY.md section 8(f) row 1)
runs on the GPU as well (``b200track/gmc.py``, csrc/b2t_gmc.cu).  ``tracker.gmc`` may be replaced by any object
with ``apply(raw_frame, detections)`` returning a 2x3 matrix."""
import numpy as np

import _b2t_path  # noqa: F401
from basetrack import BaseTrack, TrackState, STrack, BaseTracker, joint_stracks, sub_stracks, remove_duplicate_stracks  # noqa: F401
from b200track import _lib as L
from b200track import engine as _eng

import torch  # noqa: E402


class GMC:
    """``GMC(method='orb', downscale=2)`` -- what ``BoTSORT.__init__`` (reference :286) builds -- runs on the GPU estimator
    (csrc/b2t_gmc.cu through b200track/gmc.py): same key points, descriptors and matches as the reference's OpenCV calls, RANSAC
    with its own sampling sequence.  'file' and 'none' need no estimation.  'sift' and 'ecc' (unused by BoT-SORT; StrongSORT's
    ECC is outside SURVEY.md section 8) are not built and raise."""

    def __init__(self, method='orb', downscale=2, verbose=None, max_keypoints=32768):
        self.method = method
        self.downscale = max(1, int(downscale))
        self.max_keypoints = int(max_keypoints)
        self.initializedFirstFrame = False
        self._est = None
        if method == 'orb':
            pass
        elif method in ('sift', 'ecc'):
            raise NotImplementedError("GMC method %r is not built (SURVEY.md section 8f covers the ORB estimator BoT-SORT uses)" % method)
        elif method in ('file', 'files'):
            seq, ablation = verbose[0], verbose[1]
            root = 'tracker/GMC_files/MOT17_ablation' if ablation else 'tracker/GMC_files/MOTChallenge'
            for suffix in ('-FRCNN', '-DPM', '-SDP'):
                if suffix in seq:
                    seq = seq[:-len(suffix)]
            self.gmcFile = open(root + '/GMC-' + seq + '.txt', 'r')
        elif method in ('none', 'None'):
            self.method = 'none'
        else:
            raise ValueError('Error: Unknown CMC method:' + method)

    def apply(self, raw_frame, detections=None):
        if self.method == 'orb':
            return self.applyFeaures(raw_frame, detections)
        if self.method in ('file', 'files'):
            return self.applyFile(raw_frame, detections)
        return np.eye(2, 3)

    def applyFile(self, raw_frame, detections=None):
        tok = self.gmcFile.readline().split('\t')
        return np.array([[float(tok[1]), float(tok[2]), float(tok[3])],
                         [float(tok[4]), float(tok[5]), float(tok[6])]], dtype=np.float64)

    def applyFeaures(self, raw_frame, detections=None):
        """raw_frame: (H, W, 3) uint8 BGR (ndarray or tensor, host or device); detections: (n, >= 4) tlbr rows to mask out."""
        from b200track.gmc import GmcEstimator
        frame = raw_frame if isinstance(raw_frame, torch.Tensor) else torch.from_numpy(np.ascontiguousarray(raw_frame))
        h, w = int(frame.shape[0]), int(frame.shape[1])
        if self._est is None or (self._est.h, self._est.w) != (h, w):
            self._est = GmcEstimator(1, h, w, self.downscale, self.max_keypoints)
        est = self._est
        frame = frame.to(est.dev, non_blocking=True).contiguous()[None]
        dets = None
        if detections is not None and len(detections):
            d = detections if isinstance(detections, torch.Tensor) else torch.from_numpy(np.ascontiguousarray(np.asarray(detections, dtype=np.float32)))
            dets = torch.zeros((1, d.shape[0], 6), dtype=torch.float32, device=est.dev)
            dets[0, :, :4] = d[:, :4].to(est.dev)
            dets[0, :, 4] = 1.0                                   # every row handed over is masked (the caller already filtered)
        warps, stat = est.estimate(frame, dets, None, det_thresh=0.5)
        self.initializedFirstFrame = True
        H = warps[0].cpu().numpy()
        self.last_stat = stat.cpu().numpy()[0]
        if self.last_stat[5] & L.GMC_TRUNCATED and not getattr(self, '_warned', False):
            # the reference has no cap; ours keeps the first max_keypoints corners in row-major order (the top of the frame)
            print('Warning: GMC found more than %d key points; raise GMC(max_keypoints=...)' % self.max_keypoints)
            self._warned = True
        return H


def multi_gmc(stracks, H=np.eye(2, 3)):
    """Warp the Kalman state of every track in ``stracks`` (reference :250-269) on the GPU."""
    if len(stracks) == 0:
        return
    ops = _eng.ops()
    mean = ops.dev(np.asarray([st.mean.copy() for st in stracks], dtype=np.float64), torch.float64)
    cov = ops.dev(np.asarray([st.cov for st in stracks], dtype=np.float64), torch.float64)
    ops.gmc_apply(L.F64, mean, cov, H)
    mean, cov = mean.cpu().numpy(), cov.cpu().numpy()
    for st, m, c in zip(stracks, mean, cov):
        st.mean, st.cov = m, c


class BoTSORT(BaseTracker):
    _kind = 'botsort'

    def __init__(self, opts, frame_rate=30, gamma=0.02, use_GMC=True, *args, **kwargs):
        self.use_GMC = use_GMC
        super().__init__(opts, frame_rate, *args, **kwargs)
        self.use_apperance_model = False
        self.reid_model = None
        self.gamma = gamma
        self.low_conf_thresh = max(0.15, self.opts.conf_thresh - 0.3)
        self.filter_small_area = False
        self.gmc = GMC(method='orb', downscale=2, verbose=None) if use_GMC else GMC(method='none')
        self.theta_iou, self.theta_emb = 0.5, 0.25

    def _warp(self, dets, ori_img):
        if not self.use_GMC:
            return None
        det_high = dets[dets[:, 4] >= np.float32(self.det_thresh)]            # reference :380 hands over the high-score detections
        return self.gmc.apply(raw_frame=ori_img, detections=det_high)

    def get_feature(self, tlbrs, ori_img):
        """Reference :291-311: the features of the crops ``ori_img[int(y1):int(y2), int(x1):int(x2)]``, one extractor call.  The
        drop-in ``Extractor`` (or a ``ReidExtractor``) crops and runs on the device and returns a CUDA tensor; any other
        ``reid_model(list_of_crops)`` callable gets the crops as the reference cuts them."""
        if len(tlbrs) == 0:
            return np.array([])
        from reid_models.deepsort_reid import Extractor
        from b200track.reid import ReidExtractor
        net = self.reid_model.net if isinstance(self.reid_model, Extractor) else self.reid_model
        if isinstance(net, ReidExtractor):
            return net.features_from_frame(ori_img, tlbrs)
        img = ori_img.cpu().numpy() if isinstance(ori_img, torch.Tensor) else ori_img
        crops = []
        for tlbr in tlbrs:
            x1, y1, x2, y2 = list(map(int, tlbr))
            if min(x1, y1, x2, y2) < 0:                                        # the slice would wrap to the far side of the frame
                raise L.B2TError("get_feature: a box has a negative coordinate after int() (clip the boxes to the frame first)")
            crops.append(img[y1:y2, x1:x2])
        return self.reid_model(crops)

    def _step_appearance(self, det_results, ori_img, predict_only):
        """BoTSORT.update with use_apperance_model (reference :313-493): the features of exactly the reference's det_high rows
        (score >= det_thresh in float32, row order) come from ONE extractor call -- the extractor's batch-statistics BatchNorm makes a
        feature depend on the crops that share the call -- and go to the fused step row-aligned with the detections."""
        if self.reid_model is None:                                            # reference :278 builds it in the constructor
            from reid_models.deepsort_reid import Extractor
            self.reid_model = Extractor(self.opts.reid_model_path, use_cuda=True)
        self.frame_id += 1
        if predict_only:
            eng = self._get_engine(self._engine.feat_dim if self._engine is not None else 512)
            eng.set_thetas(self.theta_iou, self.theta_emb)
            return eng.step_cuda_dets([torch.zeros((0, 6), device=eng.device)], id_base=[BaseTrack._count], feats_list=None,
                                      predict_only=True)[0].copy()
        dets = self._to_numpy(det_results)
        hi = np.nonzero(dets[:, 4] >= np.float32(self.det_thresh))[0]
        feats = self.get_feature(dets[hi, :4], ori_img) if len(hi) else None
        if feats is not None:
            feats = feats if isinstance(feats, torch.Tensor) else torch.from_numpy(np.ascontiguousarray(feats, dtype=np.float32))
            if feats.dim() != 2 or feats.shape[0] != len(hi):
                raise ValueError("reid_model returned features of shape %s for %d crops" % (tuple(feats.shape), len(hi)))
        dim = int(feats.shape[1]) if feats is not None else (self._engine.feat_dim if self._engine is not None else 512)
        if dim % 32 or dim > 2048:
            raise ValueError("appearance features of length %d: the fused step takes a multiple of 32 up to 2048" % dim)
        eng = self._get_engine(dim)
        eng.set_thetas(self.theta_iou, self.theta_emb)                         # plain attributes, read every frame as the reference does
        rows = torch.zeros((len(dets), dim), dtype=torch.float32, device=eng.device)
        if feats is not None:
            rows[torch.from_numpy(hi).to(eng.device)] = feats.to(eng.device, torch.float32)
        warp = self._warp(dets, ori_img)
        return eng.step_cuda_dets([torch.from_numpy(dets).to(eng.device)], feats_list=[rows], id_base=[BaseTrack._count],
                                  warps=None if warp is None else np.asarray(warp, dtype=np.float64).reshape(1, 6))[0].copy()
