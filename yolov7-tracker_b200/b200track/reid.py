"""The appearance branch's feature extractor on the GPU (SURVEY.md section 8f row 3).

``ReidExtractor`` runs the reference's ReID network (tracker/reid_models/deepsort_reid.py:63-106 ``Net(reid=True)``: conv 3->64 + BN +
ReLU + max-pool, four stages of two ``BasicBlock``s (:14-49), 8 x 4 average pool, L2 normalisation -> 512-d unit vectors) on crops of
64 x 128 pixels: the 20 convolutions (+ folded BatchNorm + ReLU) are plans of the wgmma conv kernel (csrc/b2t_conv.cu, act = 2),
the crop / resize / normalise step, the max-pool, the residual add + ReLU and the average pool + norm are the element-wise kernels of
csrc/b2t_reid.cu.  NHWC fp16 activations, fp32 accumulation -- the same numerics as the detector branch.
``ReidExtractor.segmented`` is the same network over the det_high crops of MANY sequences in one pass, with every batch-statistics
BatchNorm normalising each sequence's crops with that sequence's statistics alone (``SegmentedReid``, used by ``TrackingPipeline``).
Weights: the ``net_dict`` of the reference's checkpoint (weights/ckpt.t7), or any state dict with the same keys.
"""
import ctypes as C

import torch

from . import _lib as L
from .conv import ConvPlan, pack_conv_weight

EPS = 1e-5                               # nn.BatchNorm2d default
STAGES = (("layer1", 64, 64, False), ("layer2", 64, 128, True), ("layer3", 128, 256, True), ("layer4", 256, 512, True))


def fold_bn(w, b, prefix, sd):
    """conv weight (Cout, Cin, k, k) [+ bias] followed by BatchNorm (eval) -> equivalent weight and bias."""
    g, beta = sd[prefix + ".weight"].double(), sd[prefix + ".bias"].double()
    mean, var = sd[prefix + ".running_mean"].double(), sd[prefix + ".running_var"].double()
    s = g / torch.sqrt(var + EPS)
    w2 = (w.double() * s[:, None, None, None]).float()
    b0 = torch.zeros_like(mean) if b is None else b.double()
    return w2, ((b0 - mean) * s + beta).float()


def folded_layers(sd):
    """The network as a list of (name, weight, bias, k, stride, relu) in execution order + the block structure."""
    convs = {}
    convs["conv0"] = fold_bn(sd["conv.0.weight"], sd["conv.0.bias"], "conv.1", sd) + (3, 1)
    for name, cin, cout, down in STAGES:
        for blk in range(2):
            p = "%s.%d" % (name, blk)
            first_down = down and blk == 0
            convs[p + ".conv1"] = fold_bn(sd[p + ".conv1.weight"], None, p + ".bn1", sd) + (3, 2 if first_down else 1)
            convs[p + ".conv2"] = fold_bn(sd[p + ".conv2.weight"], None, p + ".bn2", sd) + (3, 1)
            if (p + ".downsample.0.weight") in sd:
                convs[p + ".down"] = fold_bn(sd[p + ".downsample.0.weight"], None, p + ".downsample.1", sd) + (1, 2 if first_down else 1)
    return convs


def raw_layers(sd):
    """The same layers WITHOUT folding: (weight, bias or zeros, k, stride, gamma, beta) -- for BatchNorm with batch statistics."""
    convs = {}

    def one(wk, bk, bn, k, s):
        w = sd[wk]
        b = sd[bk] if bk else torch.zeros(w.shape[0])
        return (w, b, k, s, sd[bn + ".weight"], sd[bn + ".bias"])
    convs["conv0"] = one("conv.0.weight", "conv.0.bias", "conv.1", 3, 1)
    for name, cin, cout, down in STAGES:
        for blk in range(2):
            p = "%s.%d" % (name, blk)
            s = 2 if (down and blk == 0) else 1
            convs[p + ".conv1"] = one(p + ".conv1.weight", None, p + ".bn1", 3, s)
            convs[p + ".conv2"] = one(p + ".conv2.weight", None, p + ".bn2", 3, 1)
            if (p + ".downsample.0.weight") in sd:
                convs[p + ".down"] = one(p + ".downsample.0.weight", None, p + ".downsample.1", 1, s)
    return convs


class ReidExtractor:
    def __init__(self, state_dict, device="cuda:0", dtype=torch.float16, bn_mode="batch"):
        """bn_mode: "batch" -- what the reference computes: its extractor is never switched to eval() (deepsort_reid.py:112-121), so
        BatchNorm normalises each call with that call's batch statistics (features depend on which crops share the call); "running" --
        eval-mode BatchNorm (running statistics), folded into the convolutions: one fused conv + bias + ReLU launch per layer."""
        if bn_mode not in ("batch", "running"):
            raise ValueError("bn_mode must be 'batch' or 'running'")
        self.bn_mode = bn_mode
        if not torch.cuda.is_available():
            raise L.B2TError("ReidExtractor needs a CUDA device (there is no CPU fallback)")
        self.lib = L.load()
        self.dev = torch.device(device)
        self.dtype = dtype
        self.code = L.act_dtype_code(dtype)
        sd = {k: v.detach().to("cpu", torch.float32) for k, v in state_dict.items() if v.dtype.is_floating_point}
        self.weights, self.bn = {}, {}
        layers = folded_layers(sd) if bn_mode == "running" else raw_layers(sd)
        for name, item in layers.items():
            w, b, k, s = item[:4]
            cin_pad = 16 if w.shape[1] == 3 else None
            self.weights[name] = (pack_conv_weight(w.to(self.dev), cin_pad=cin_pad, dtype=dtype), b.to(self.dev).float().contiguous(), w.shape[0], w.shape[1] if cin_pad is None else 16, k, s)
            if bn_mode == "batch":
                self.bn[name] = (item[4].to(self.dev).float().contiguous(), item[5].to(self.dev).float().contiguous())
        self._nets = {}

    def _stream(self):
        return C.c_void_p(torch.cuda.current_stream(self.dev).cuda_stream)

    def _build(self, n, seg=None):
        """Buffers and conv plans for a batch of n crops.  seg (a SegmentedReid): BatchNorm statistics per segment of seg.offsets and
        the pooled features of crop j to row seg.rowmap[j] of seg.feats."""
        dev, dt = self.dev, self.dtype
        buf = lambda h, w, c: torch.zeros((n, h, w, c), dtype=dt, device=dev)          # noqa: E731
        net = {"n": n, "valid": n, "x": buf(128, 64, 16), "c0": buf(128, 64, 64), "ops": []}
        ops = net["ops"]
        bn_ws = [None]                         # BatchNorm scratch, sized below for the largest layer of this capacity
        bn_bytes = [0]

        def check(rc):
            if rc != 0:
                raise L.B2TError("libb200track error %d: %s" % (rc, (self.lib.b2t_detect_last_error() or b"").decode()))

        def conv(name, x, y, h, w, act):
            """act: 2 = ReLU after the (folded or batch-statistics) BatchNorm, 0 = none."""
            wp, b, cout, cin, k, s = self.weights[name]
            batch = self.bn_mode == "batch"
            plan = ConvPlan(x, wp, b, y, n, h, w, cin, 0, cout, k, s, 0, act=0 if batch else act)
            ops.append(plan.run)
            if batch:
                g, beta = self.bn[name]
                ho, wo = h // s, w // s
                if seg is not None:
                    bn_bytes[0] = max(bn_bytes[0], int(self.lib.b2t_batchnorm_segments_workspace_bytes(seg.S, n, ho * wo, cout)))
                    # statistics per sequence (segment), the padding crops past offsets[S] excluded
                    ops.append(lambda y=y, g=g, beta=beta, c=cout, hw=ho * wo, relu=int(act == 2): check(self.lib.b2t_batchnorm_batch_stats_segments(
                        y.data_ptr(), y.data_ptr(), seg.offsets.data_ptr(), seg.S, n, hw, c, g.data_ptr(), beta.data_ptr(), EPS, relu,
                        bn_ws[0].data_ptr(), self.code, self._stream())))
                    return plan
                bn_bytes[0] = max(bn_bytes[0], int(self.lib.b2t_batchnorm_workspace_bytes(n * ho * wo, cout)))     # grows with n_pix
                # statistics over the VALID crops only (net["valid"]): the rows that pad the batch to its capacity must not count
                ops.append(lambda y=y, g=g, beta=beta, c=cout, hw=ho * wo, relu=int(act == 2): check(self.lib.b2t_batchnorm_batch_stats(
                    y.data_ptr(), y.data_ptr(), net["valid"] * hw, c, g.data_ptr(), beta.data_ptr(), EPS, relu, bn_ws[0].data_ptr(), self.code, self._stream())))
            return plan
        net["plans"] = [conv("conv0", net["x"], net["c0"], 128, 64, 2)]
        cur = buf(64, 32, 64)
        c0 = net["c0"]
        ops.append(lambda a=c0, o=cur: check(self.lib.b2t_maxpool3x3s2(a.data_ptr(), o.data_ptr(), n, 128, 64, 64, self.code, self._stream())))
        h, w = 64, 32
        for name, cin, cout, down in STAGES:
            for blk in range(2):
                p = "%s.%d" % (name, blk)
                s = 2 if (down and blk == 0) else 1
                ho, wo = h // s, w // s
                y1, y2, out = buf(ho, wo, cout), buf(ho, wo, cout), buf(ho, wo, cout)
                net["plans"].append(conv(p + ".conv1", cur, y1, h, w, 2))
                net["plans"].append(conv(p + ".conv2", y1, y2, ho, wo, 0))
                skip = cur
                if (p + ".down") in self.weights:
                    skip = buf(ho, wo, cout)
                    net["plans"].append(conv(p + ".down", cur, skip, h, w, 0))
                ops.append(lambda a=skip, b=y2, o=out: check(self.lib.b2t_add_relu(a.data_ptr(), b.data_ptr(), o.data_ptr(), a.numel(), self.code, self._stream())))
                net.setdefault("keep", []).extend([y1, y2, skip, out])
                cur, h, w = out, ho, wo
        if self.bn_mode == "batch":
            bn_ws[0] = net["bn_ws"] = torch.zeros((bn_bytes[0] + 7) // 8, dtype=torch.float64, device=dev)
        last = cur
        if seg is not None:
            ops.append(lambda a=last: check(self.lib.b2t_avgpool_l2norm_rows(a.data_ptr(), seg.feats.data_ptr(), seg.rowmap.data_ptr(), n, h * w, 512,
                                                                              self.code, self._stream())))
        else:
            net["feat"] = torch.zeros((n, 512), dtype=torch.float32, device=dev)
            ops.append(lambda a=last, o=net["feat"]: check(self.lib.b2t_avgpool_l2norm(a.data_ptr(), o.data_ptr(), n, h * w, 512, self.code, self._stream())))
        net["flops"] = sum(p.flops for p in net["plans"])
        net["launches"] = len(ops) + 1
        return net

    def _net(self, n):
        cap = 32
        while cap < n:
            cap *= 2
        if cap not in self._nets:
            with torch.cuda.device(self.dev):
                self._nets[cap] = self._build(cap)
        return self._nets[cap]

    def segmented(self, n_seq, dmax, cap=None):
        """The network over the det_high crops of n_seq sequences at once, at a fixed capacity of cap crops (default n_seq * dmax,
        which cannot overflow): see SegmentedReid."""
        return SegmentedReid(self, n_seq, dmax, n_seq * dmax if cap is None else cap)

    def features_segments(self, frames, tlbrs_per_seq, cap=None):
        """Host-facing form of the segmented pass (tests, tools): frames (S, H, W, 3) uint8 BGR, tlbrs_per_seq: per sequence an
        (n_s, 4) array of boxes.  Returns per sequence the (n_s, 512) features -- each sequence's crops normalised with its own batch
        statistics, as ``features_from_frame(frames[s], tlbrs_per_seq[s])`` alone computes them.  Raises B2TError for a refused crop."""
        import numpy as np
        f = frames if isinstance(frames, torch.Tensor) else torch.from_numpy(np.ascontiguousarray(frames))
        f = f.to(self.dev).contiguous()
        S = int(f.shape[0])
        if len(tlbrs_per_seq) != S:
            raise L.B2TError("features_segments: %d box lists for %d frames" % (len(tlbrs_per_seq), S))
        boxes = [np.asarray(t, dtype=np.float32).reshape(-1, 4) for t in tlbrs_per_seq]
        dmax = max(1, max(len(b) for b in boxes))
        dets = np.zeros((S, dmax, 6), np.float32)
        for s, b in enumerate(boxes):
            dets[s, :len(b), :4] = b
            dets[s, :len(b), 4] = 1.0
        seg = self.segmented(S, dmax, cap)
        d_dets = torch.from_numpy(dets).to(self.dev)
        d_cnt = torch.tensor([len(b) for b in boxes], dtype=torch.int32, device=self.dev)
        with torch.cuda.device(self.dev):
            seg.cut(f, d_dets, d_cnt, 0.5)
            seg.run()
            status = seg.status.cpu().numpy()
        seg.raise_for_status(status)
        return [seg.feats[s, :len(b)].clone() for s, b in enumerate(boxes)]

    def features(self, pixels, crops):
        """pixels: uint8 device tensor holding BGR pixels (a batch of frames, or crops packed back to back); crops: (n, 4) int64 rows
        {byte offset of the crop's first pixel, row pitch in bytes, height, width}.  Returns (n, 512) float32 unit vectors (device)."""
        n = int(crops.shape[0])
        if n == 0:
            return torch.zeros((0, 512), dtype=torch.float32, device=self.dev)
        net = self._net(n)
        net["valid"] = n
        cr = torch.zeros((net["n"], 4), dtype=torch.int64, device=self.dev)
        cr[:] = crops[0].to(self.dev)                           # unused rows repeat a valid crop
        cr[:n] = crops.to(self.dev)
        with torch.cuda.device(self.dev):
            rc = self.lib.b2t_reid_crops(pixels.data_ptr(), cr.data_ptr(), net["n"], net["x"].data_ptr(), self.code, self._stream())
            if rc != 0:
                raise L.B2TError("b2t_reid_crops: %s" % (self.lib.b2t_detect_last_error() or b"").decode())
            for op in net["ops"]:
                op()
        self.last_net = net
        return net["feat"][:n]

    def features_from_frame(self, frame, tlbrs):
        """BoTSORT.get_feature (botsort.py:291-311): frame (H, W, 3) uint8 BGR tensor / array, tlbrs (n, 4): the crops are
        ``ori_img[int(y1):int(y2), int(x1):int(x2)]``."""
        import numpy as np
        f = frame if isinstance(frame, torch.Tensor) else torch.from_numpy(np.ascontiguousarray(frame))
        f = f.to(self.dev).contiguous()
        H, W = int(f.shape[0]), int(f.shape[1])
        t = np.asarray(tlbrs, dtype=np.float64).reshape(-1, 4).astype(np.int64)                 # list(map(int, tlbr)): truncation
        if (t < 0).any():
            # ori_img[int(y1):int(y2), int(x1):int(x2)] would wrap a negative index to the far side of the frame
            raise L.B2TError("ReidExtractor: a box has a negative coordinate after int() (clip the boxes to the frame first)")
        x1, y1 = np.clip(t[:, 0], 0, W), np.clip(t[:, 1], 0, H)
        x2, y2 = np.clip(t[:, 2], 0, W), np.clip(t[:, 3], 0, H)
        if ((x2 - x1) < 1).any() or ((y2 - y1) < 1).any():
            raise L.B2TError("ReidExtractor: a crop has zero size (the reference prints 'size in bbox exists zero' and exits)")
        crops = torch.from_numpy(np.stack([(y1 * W + x1) * 3, np.full_like(x1, 3 * W), y2 - y1, x2 - x1], 1))
        return self.features(f, crops)

    def __call__(self, im_crops):
        """Extractor.__call__ (:148-153): a list of (h, w, 3) uint8 BGR arrays -> (n, 512) float32 ndarray on the host."""
        import numpy as np
        if len(im_crops) == 0:
            return np.zeros((0, 512), np.float32)
        offs, rows, o = [], [], 0
        for im in im_crops:
            h, w = int(im.shape[0]), int(im.shape[1])
            if h < 1 or w < 1:
                raise L.B2TError("ReidExtractor: a crop has zero size (the reference prints 'size in bbox exists zero' and exits)")
            rows.append((o, 3 * w, h, w))
            offs.append(np.ascontiguousarray(im, dtype=np.uint8).reshape(-1))
            o += h * w * 3
        pixels = torch.from_numpy(np.concatenate(offs)).to(self.dev)
        return self.features(pixels, torch.tensor(rows, dtype=torch.int64)).cpu().numpy()


class SegmentedReid:
    """The extractor over the det_high crops of S sequences in ONE pass, at a fixed capacity of `cap` crops, with nothing in a step that
    depends on a host-side count: the crop descriptors, segment offsets and row map are device tensors written by
    b2t_reid_crops_from_dets from the NMS output.  ``cut`` (two launches) builds the crop list and cuts the crops out of the frames, after
    which the frame buffer may be overwritten; ``run`` replays one CUDA graph of the 20 convs, the BatchNorms (statistics per sequence in
    batch mode, b2t_batchnorm_batch_stats_segments; folded in running mode), pools and adds, and writes the features of crop j to row
    rowmap[j] of ``feats`` (S, dmax, 512) -- the tensor TrackEngine.step_device(feats=) takes.  Padding crops cost full compute and go
    nowhere."""

    def __init__(self, ext, n_seq, dmax, cap):
        if n_seq < 1 or dmax < 1 or cap < 1:
            raise L.B2TError("SegmentedReid: n_seq, dmax and cap must be >= 1 (got %d, %d, %d)" % (n_seq, dmax, cap))
        self.ext, self.S, self.dmax, self.cap = ext, int(n_seq), int(dmax), int(cap)
        dev = ext.dev
        with torch.cuda.device(dev):
            self.crops = torch.zeros((self.cap, 4), dtype=torch.int64, device=dev)
            self.offsets = torch.zeros(self.S + 1, dtype=torch.int32, device=dev)
            self.rowmap = torch.full((self.cap,), -1, dtype=torch.int32, device=dev)
            self.status = torch.zeros(self.S + 1, dtype=torch.int32, device=dev)
            self.feats = torch.zeros((self.S, self.dmax, 512), dtype=torch.float32, device=dev)
            self.net = ext._build(self.cap, seg=self)
        self.graph = None
        self.bytes = sum(t.numel() * t.element_size() for t in self._tensors())

    def _tensors(self):
        net = self.net
        ts = [self.crops, self.offsets, self.rowmap, self.status, self.feats, net["x"], net["c0"]] + net.get("keep", [])
        if "bn_ws" in net:
            ts.append(net["bn_ws"])
        seen, out = set(), []
        for t in ts:
            if t.data_ptr() not in seen:
                seen.add(t.data_ptr()); out.append(t)
        return out

    def cut(self, frames, dets, det_count, det_thresh):
        """On the current stream: frames (S, H, W, 3) uint8 device tensor, dets (S, dmax, 6) float32, det_count (S,) int32 (the
        detector's out / out_count); det_thresh: the tracker's conf_thresh (compared in float32)."""
        ext = self.ext
        if tuple(dets.shape) != (self.S, self.dmax, 6) or dets.dtype != torch.float32 or det_count.dtype != torch.int32 or tuple(det_count.shape) != (self.S,):
            raise L.B2TError("SegmentedReid.cut: dets must be float32 (%d, %d, 6) and det_count int32 (%d,)" % (self.S, self.dmax, self.S))
        if frames.dtype != torch.uint8 or frames.dim() != 4 or int(frames.shape[0]) != self.S or int(frames.shape[3]) != 3 or not frames.is_contiguous():
            raise L.B2TError("SegmentedReid.cut: frames must be a contiguous uint8 (%d, H, W, 3) tensor" % self.S)
        H, W = int(frames.shape[1]), int(frames.shape[2])
        rc = ext.lib.b2t_reid_crops_from_dets(dets.data_ptr(), det_count.data_ptr(), self.S, self.dmax, float(det_thresh), H, W, self.cap,
                                              self.crops.data_ptr(), self.offsets.data_ptr(), self.rowmap.data_ptr(), self.status.data_ptr(), ext._stream())
        if rc == 0:
            rc = ext.lib.b2t_reid_crops(frames.data_ptr(), self.crops.data_ptr(), self.cap, self.net["x"].data_ptr(), ext.code, ext._stream())
        if rc != 0:
            raise L.B2TError("SegmentedReid.cut: %s" % (ext.lib.b2t_detect_last_error() or b"").decode())

    def run(self):
        """On the current stream: the network on the cut crops -> feats (one CUDA graph; captured on the first call)."""
        if self.graph is None:
            self.capture()
        self.graph.replay()

    def capture(self):
        """Capture the graph of ``run`` (synchronises the device).  The ops read only device tensors, so capturing before any ``cut``
        is safe: the warm-up normalises nothing (empty segments) and writes no feature row (row map all -1)."""
        cur = torch.cuda.current_stream(self.ext.dev)
        cs = torch.cuda.Stream(device=self.ext.dev)              # captured on a side stream (the current one may be the legacy default)
        cs.wait_stream(cur)
        with torch.cuda.device(self.ext.dev), torch.cuda.stream(cs):
            for op in self.net["ops"]:                           # warm-up outside the capture (module loading)
                op()
        cs.synchronize()
        self.graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(self.graph, stream=cs):
            for op in self.net["ops"]:
                op()
        cur.wait_stream(cs)

    def raise_for_status(self, status):
        """status: the (S + 1,) status words read back (host array) -> B2TError naming the first refused condition and sequence."""
        for s in range(self.S):
            bits = int(status[s])
            if bits & L.REID_OVERFLOW:
                raise L.B2TError("ReID: sequence %d: the det_high crops of this step (%d in all sequences) exceed reid_cap = %d" % (s, int(status[self.S]), self.cap))
            if bits & L.REID_ZERO_SIZE:
                raise L.B2TError("ReID: sequence %d: a det_high box gives a crop of zero size (the reference prints 'size in bbox exists zero' and exits)" % s)
            if bits & L.REID_NEGATIVE:
                raise L.B2TError("ReID: sequence %d: a det_high box has a negative coordinate after int() (the reference's slice would wrap)" % s)
