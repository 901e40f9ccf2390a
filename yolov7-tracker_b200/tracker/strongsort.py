"""Drop-in for the reference's ``tracker/strongsort.py``: ``StrongSORT(opts, frame_rate=30, gamma=0.1, use_ECC=True, use_AFLink=True,
use_GSI=True, num_of_budget=20)``, so that ``track.py --tracker strongsort`` runs unchanged.

``StrongSORT.update`` (reference :91-250) runs as one call of the fused step's StrongSORT kind (csrc/b2t_step.cuh, B2T_STRONGSORT):
the feature distances, the dense gamma * IoU + (1 - gamma) * Euclidean cost of associations 1 and 3, association 2, the q18 marking,
births and the list algebra.  The appearance features come from the drop-in ``osnet_x0_25`` on the device (``get_feature`` cuts the
crops of the rows with score > det_thresh out of the frame, ``OsnetExtractor.features_from_frame``), the camera motion from
``GMC('ecc')`` on the device; neither leaves the device before the step.  ``update`` / ``update_without_detection`` return the same
live track views as the drop-in ``BoTSORT`` (``tlwh``, ``track_id``, ``cls``, ``features``).  ``use_AFLink`` / ``use_GSI`` are
accepted and do nothing, as in the reference (its TODOs)."""
import numpy as np
import torch

import _b2t_path  # noqa: F401
from basetrack import BaseTrack, TrackState, STrack, BaseTracker, joint_stracks, sub_stracks, remove_duplicate_stracks  # noqa: F401
from reid_models.OSNet import osnet_x0_25
from reid_models.load_model_tools import load_pretrained_weights
from botsort import GMC, multi_gmc  # noqa: F401
from b200track import _lib as L


class StrongSORT(BaseTracker):
    _kind = 'strongsort'

    def __init__(self, opts, frame_rate=30, gamma=0.1, use_ECC=True, use_AFLink=True, use_GSI=True, num_of_budget=20, *args, **kwargs):
        super().__init__(opts, frame_rate, *args, **kwargs)
        self.gamma = gamma
        self.reid_model = osnet_x0_25(num_classes=1, pretrained=False)
        self.reid_model.cuda().eval()
        load_pretrained_weights(self.reid_model, opts.reid_model_path)
        self.use_ECC = use_ECC
        self.ECC = GMC(method='ecc', downscale=2, verbose=None)
        self.use_AFLink = use_AFLink
        self.use_GSI = use_GSI
        self.matching_thresh = min(0.3, self.opts.iou_thresh - 0.2)
        self.num_of_budget = num_of_budget

    def get_feature(self, tlbrs, ori_img):
        """Reference :66-89: the OSNet features of the crops ``ori_img[int(y1):int(y2), int(x1):int(x2)]``, resized to 128 x 256, cut
        and computed on the device.  A negative coordinate after int() or an empty crop raises B2TError."""
        dev = next(self.reid_model.parameters()).device
        return self.reid_model.extractor(dev, (128, 256)).features_from_frame(ori_img, tlbrs)

    def _get_engine(self, feat_dim=0):
        if self._engine is None:
            from b200track.engine import TrackEngine
            self._engine = TrackEngine(kind='strongsort', n_seq=1, kalman_format=self.opts.kalman_format, conf_thresh=self.opts.conf_thresh,
                                       track_buffer=self.opts.track_buffer, frame_rate=self._frame_rate, use_gmc=bool(self.use_ECC),
                                       feat_dim=feat_dim, gamma=self.gamma, **self._engine_kw)
        if self._engine.feat_dim != feat_dim:
            raise RuntimeError("StrongSORT started with features of length %d and now gets %d" % (self._engine.feat_dim, feat_dim))
        return self._engine

    def _step(self, det_results, ori_img, predict_only=False):
        self.frame_id += 1
        if predict_only:                                                       # BaseTracker.update_without_detection: no ECC
            eng = self._get_engine(self._engine.feat_dim if self._engine is not None else 512)
            rows = eng.step_cuda_dets([torch.zeros((0, 6), device=eng.device)], id_base=[BaseTrack._count], feats_list=None,
                                      predict_only=True)[0]
            return self._finish_step(rows, True)
        dets = self._to_numpy(det_results)
        sel = np.nonzero(dets[:, 4] > np.float32(self.det_thresh))[0]          # reference :118, float32 compare
        feats = self.get_feature(dets[sel, :4], ori_img) if len(sel) else None
        if feats is not None:
            feats = feats if isinstance(feats, torch.Tensor) else torch.from_numpy(np.ascontiguousarray(feats, dtype=np.float32))
            if feats.dim() != 2 or feats.shape[0] != len(sel):
                raise ValueError("get_feature returned features of shape %s for %d crops" % (tuple(feats.shape), len(sel)))
        dim = int(feats.shape[1]) if feats is not None else (self._engine.feat_dim if self._engine is not None else 512)
        eng = self._get_engine(dim)
        rows = torch.zeros((len(dets), dim), dtype=torch.float32, device=eng.device)
        if feats is not None:
            rows[torch.from_numpy(sel).to(eng.device)] = feats.to(eng.device, torch.float32)
        warp = self.ECC.apply(raw_frame=ori_img, detections=None) if self.use_ECC else None     # reference :140-144
        out = eng.step_cuda_dets([torch.from_numpy(dets).to(eng.device)], feats_list=[rows], id_base=[BaseTrack._count],
                                 warps=None if warp is None else np.asarray(warp, dtype=np.float64).reshape(1, 6))[0]
        return self._finish_step(out)
