"""StrongSORT's appearance network on the GPU: OSNet x0.25 (tracker/strongsort.py:26-29, :47-89, tracker/reid_models/OSNet.py) on
the kernels of csrc/b2t_osnet.cu.

``OsnetExtractor`` folds the eval-mode BatchNorms of an ``osnet_x0_25`` state dict into float32 weights (in float64) and runs the
network on NHWC 16-bit activations with fp32 accumulation: crop / resize / normalise, the fused stem (7 x 7 conv + max-pool), per
OSBlock one 1 x 1, ten fused LightConv3x3, the shared channel gate summed over the four streams, and conv3 + the identity branch in
one 1 x 1 launch; the transitions' AvgPool is fused into their 1 x 1, and the head pools, applies fc + BatchNorm1d + ReLU and writes
(n, 512) float32 -- the reference's unnormalised features.  Batches run at a capacity of the next power of two >= 32, one CUDA graph
per capacity; every kernel computes a crop from that crop's data alone in a fixed order, so a crop's feature does not depend on the
batch, its position in it or the capacity.
"""
import ctypes as C

import numpy as np
import torch

from . import _lib as L

EPS = 1e-5
STAGES = (("conv2", 16, 64, True), ("conv3", 64, 96, True), ("conv4", 96, 128, False))
STREAMS = (("conv2a", 1), ("conv2b", 2), ("conv2c", 3), ("conv2d", 4))
FEATURE_DIM = 512


def _bn_scale_shift(sd, p):
    g, b = sd[p + ".weight"].double(), sd[p + ".bias"].double()
    mean, var = sd[p + ".running_mean"].double(), sd[p + ".running_var"].double()
    s = g / torch.sqrt(var + EPS)
    return s, b - mean * s


def _conv_bn(sd, p):
    """Conv (no bias) + BatchNorm -> (weight [cin * k * k][cout] float64 with the scale folded, bias [cout])"""
    s, t = _bn_scale_shift(sd, p + ".bn")
    w = sd[p + ".conv.weight"].double() * s[:, None, None, None]
    return w, t


def _light(sd, p):
    """LightConv3x3 -> (w1 [ci][co], dw [9][c] with the BN scale folded, bias [c])"""
    s, t = _bn_scale_shift(sd, p + ".bn")
    w1 = sd[p + ".conv1.weight"].double()[:, :, 0, 0].t()
    dw = (sd[p + ".conv2.weight"].double()[:, 0] * s[:, None, None]).permute(1, 2, 0).reshape(9, -1)
    return w1, dw, t


def fold(sd):
    """The network's float32 weights in the layouts the kernels read (float64 folding), keyed by layer."""
    f = {}
    w, b = _conv_bn(sd, "conv1")
    f["stem"] = (w.permute(2, 3, 1, 0).reshape(147, 16), b)
    for stage, cin, cout, trans in STAGES:
        for blk in range(2):
            p = "%s.%d" % (stage, blk)
            w, b = _conv_bn(sd, p + ".conv1")
            f[p + ".conv1"] = (w[:, :, 0, 0].t(), b)
            for name, k in STREAMS:
                for i in range(k):
                    q = ("%s.%s" % (p, name)) if k == 1 else ("%s.%s.%d" % (p, name, i))
                    f[q] = _light(sd, q)
            f[p + ".gate"] = tuple(sd[p + ".gate." + n].double().reshape(sd[p + ".gate." + n].shape[0], -1).squeeze(-1) if n.endswith("bias")
                                   else sd[p + ".gate." + n].double()[:, :, 0, 0] for n in ("fc1.weight", "fc1.bias", "fc2.weight", "fc2.bias"))
            w3, b3 = _conv_bn(sd, p + ".conv3")
            if (p + ".downsample.conv.weight") in sd:
                wd, bd = _conv_bn(sd, p + ".downsample")
                f[p + ".conv3"] = (torch.cat([w3[:, :, 0, 0].t(), wd[:, :, 0, 0].t()], 0), b3 + bd)
            else:
                f[p + ".conv3"] = (w3[:, :, 0, 0].t(), b3)
        if trans:
            w, b = _conv_bn(sd, "%s.2.0" % stage)
            f[stage + ".trans"] = (w[:, :, 0, 0].t(), b)
    w, b = _conv_bn(sd, "conv5")
    f["conv5"] = (w[:, :, 0, 0].t(), b)
    s, t = _bn_scale_shift(sd, "fc.1")
    f["head"] = ((sd["fc.0.weight"].double() * s[:, None]).t(), sd["fc.0.bias"].double() * s + t)
    return {k: tuple(a.float().contiguous() for a in v) for k, v in f.items()}


class OsnetExtractor:
    def __init__(self, state_dict, device="cuda:0", dtype=torch.float16, size=(128, 256)):
        """state_dict: an osnet_x0_25 state dict (the ``module.`` prefix of a DataParallel checkpoint is stripped; the classifier is
        not used).  size: (rows, columns) of the network input, multiples of 16; (128, 256) is what StrongSORT feeds
        (cv2.resize(dsize=(256, 128)) gives 128 rows x 256 columns)."""
        if not torch.cuda.is_available():
            raise L.B2TError("OsnetExtractor needs a CUDA device (there is no CPU fallback)")
        h, w = int(size[0]), int(size[1])
        if h < 16 or w < 16 or h % 16 or w % 16:
            raise L.B2TError("OsnetExtractor: size must be (rows, columns), multiples of 16, got %r" % (tuple(size),))
        self.size = (h, w)
        self.lib = L.load()
        self.dev = torch.device(device)
        self.dtype = dtype
        self.code = L.act_dtype_code(dtype)
        sd = {(k[7:] if k.startswith("module.") else k): v.detach().to("cpu") for k, v in state_dict.items()}
        sd = {k: v.double() for k, v in sd.items() if v.is_floating_point()}
        if tuple(sd.get("conv1.conv.weight", torch.zeros(0)).shape) != (16, 3, 7, 7) or tuple(sd.get("fc.0.weight", torch.zeros(0)).shape) != (512, 128):
            raise L.B2TError("OsnetExtractor: not an osnet_x0_25 state dict (conv1.conv.weight must be 16 x 3 x 7 x 7, fc.0.weight 512 x 128)")
        try:
            folded = fold(sd)
        except KeyError as e:
            raise L.B2TError("OsnetExtractor: the state dict lacks %s" % e) from None
        self.w = {k: tuple(a.to(self.dev) for a in v) for k, v in folded.items()}
        self._nets = {}

    def _stream(self):
        return C.c_void_p(torch.cuda.current_stream(self.dev).cuda_stream)

    def _check(self, rc, what):
        if rc != 0:
            raise L.B2TError("%s: %s" % (what, (self.lib.b2t_detect_last_error() or b"").decode()))

    def _build(self, n):
        """Buffers and the launch list of the network at capacity n (everything after the input buffer)."""
        lib, dev, dt, code = self.lib, self.dev, self.dtype, self.code
        H, W = self.size
        buf = lambda h, w, c: torch.zeros((n, h, w, c), dtype=dt, device=dev)          # noqa: E731
        net = {"n": n, "x4": buf(H, W, 4), "feat": torch.zeros((n, FEATURE_DIM), dtype=torch.float32, device=dev)}
        ops, keep, kernels = [], [], []          # kernels: (kind, FLOP, bytes moved) per launch, from the shapes
        P = lambda t: C.c_void_p(t.data_ptr())                                           # noqa: E731
        ck = self._check

        def add(name, fn, flop, nbytes):
            kernels.append((name, float(flop), float(nbytes)))
            ops.append(fn)

        h, w = H // 4, W // 4
        stem_out = buf(h, w, 16)
        keep.append(stem_out)
        sw, sb = self.w["stem"]
        net["stem_in"] = "x4"
        add("stem", lambda: ck(lib.b2t_osnet_stem(P(net[net["stem_in"]]), 4 if net["stem_in"] == "x4" else 16, P(sw), P(sb), n, H, W, P(stem_out),
                                                  code, self._stream()), "b2t_osnet_stem"),
            2 * n * (H // 2) * (W // 2) * 16 * 147, 2 * n * (H * W * 4 + h * w * 16))
        cur, c = stem_out, 16
        for stage, cin, cout, trans in STAGES:
            mid = cout // 4
            x1, x2, t1, t2 = buf(h, w, mid), buf(h, w, mid), buf(h, w, mid), buf(h, w, mid)
            ss = [buf(h, w, mid) for _ in range(4)]
            outs = [buf(h, w, cout), buf(h, w, cout)]
            keep += [x1, x2, t1, t2] + ss + outs
            for blk in range(2):
                p = "%s.%d" % (stage, blk)
                wt, b = self.w[p + ".conv1"]
                add("pointwise", lambda x=cur, ci=c, wt=wt, b=b, y=x1, h=h, w=w, co=mid: ck(lib.b2t_osnet_pointwise(
                    P(x), ci, None, 0, P(wt), P(b), None, P(y), n, h, w, co, 1, 0, code, self._stream()), "b2t_osnet_pointwise"),
                    2 * n * h * w * c * mid, 2 * n * h * w * (c + mid))
                for (name, k), dst in zip(STREAMS, ss):
                    src = x1
                    for i in range(k):
                        q = ("%s.%s" % (p, name)) if k == 1 else ("%s.%s.%d" % (p, name, i))
                        y = dst if i == k - 1 else (t1 if src is not t1 else t2)
                        w1, dw, lb = self.w[q]
                        add("lightconv", lambda x=src, y=y, w1=w1, dw=dw, lb=lb, h=h, w=w, c=mid: ck(lib.b2t_osnet_lightconv(
                            P(x), P(w1), P(dw), P(lb), P(y), n, h, w, c, code, self._stream()), "b2t_osnet_lightconv"),
                            2 * n * h * w * (mid * mid + 9 * mid), 2 * n * h * w * 2 * mid)
                        src = y
                g1w, g1b, g2w, g2b = self.w[p + ".gate"]
                add("gate_sum", lambda g=(g1w, g1b, g2w, g2b), ss=ss, y=x2, h=h, w=w, c=mid: ck(lib.b2t_osnet_gate_sum(
                    P(ss[0]), P(ss[1]), P(ss[2]), P(ss[3]), P(g[0]), P(g[1]), P(g[2]), P(g[3]), P(y), n, h * w, c, int(g[0].shape[0]),
                    code, self._stream()), "b2t_osnet_gate_sum"), 4 * n * h * w * mid * 3, 2 * n * h * w * mid * 9)
                wt, b = self.w[p + ".conv3"]
                out = outs[blk]
                if c != cout:          # downsample branch: one accumulator over [x2, x]
                    add("pointwise", lambda x=cur, ci=c, wt=wt, b=b, y=out, x2=x2, m=mid, co=cout, h=h, w=w: ck(lib.b2t_osnet_pointwise(
                        P(x2), m, P(x), ci, P(wt), P(b), None, P(y), n, h, w, co, 1, 0, code, self._stream()), "b2t_osnet_pointwise"),
                        2 * n * h * w * (mid + c) * cout, 2 * n * h * w * (mid + c + cout))
                else:                  # identity added before the ReLU
                    add("pointwise", lambda x=cur, wt=wt, b=b, y=out, x2=x2, m=mid, co=cout, h=h, w=w: ck(lib.b2t_osnet_pointwise(
                        P(x2), m, None, 0, P(wt), P(b), P(x), P(y), n, h, w, co, 1, 0, code, self._stream()), "b2t_osnet_pointwise"),
                        2 * n * h * w * mid * cout, 2 * n * h * w * (mid + 2 * cout))
                cur, c = out, cout
            if trans:
                wt, b = self.w[stage + ".trans"]
                pooled = buf(h // 2, w // 2, cout)
                keep.append(pooled)
                add("pointwise_pool", lambda x=cur, wt=wt, b=b, y=pooled, co=cout, h=h, w=w: ck(lib.b2t_osnet_pointwise(
                    P(x), co, None, 0, P(wt), P(b), None, P(y), n, h, w, co, 1, 1, code, self._stream()), "b2t_osnet_pointwise"),
                    2 * n * h * w * cout * cout, 2 * n * h * w * cout * 5 // 4)
                cur, h, w = pooled, h // 2, w // 2
        wt, b = self.w["conv5"]
        c5 = buf(h, w, 128)
        keep.append(c5)
        add("pointwise", lambda x=cur, wt=wt, b=b, h=h, w=w: ck(lib.b2t_osnet_pointwise(P(x), 128, None, 0, P(wt), P(b), None, P(c5), n, h, w, 128, 1,
                                                                                      0, code, self._stream()), "b2t_osnet_pointwise"),
            2 * n * h * w * 128 * 128, 2 * n * h * w * 256)
        hw_, hb = self.w["head"]
        add("head", lambda hw=h * w: ck(lib.b2t_osnet_head(P(c5), P(hw_), P(hb), P(net["feat"]), n, hw, 128, FEATURE_DIM, code, self._stream()),
                                       "b2t_osnet_head"), 2 * n * (h * w * 128 + 128 * FEATURE_DIM), n * (2 * h * w * 128 + 4 * FEATURE_DIM))
        net["ops"], net["keep"], net["kernels"], net["graphs"] = ops, keep, kernels, {}
        return net

    def _net(self, n):
        cap = 32
        while cap < n:
            cap *= 2
        if cap not in self._nets:
            with torch.cuda.device(self.dev):
                self._nets[cap] = self._build(cap)
        return self._nets[cap]

    def _run(self, net, stem_in):
        """The network from net[stem_in] ("x4": crops, "x16": an NCHW image batch) -> net["feat"]; one CUDA graph per input kind."""
        net["stem_in"] = stem_in
        g = net["graphs"].get(stem_in)
        if g is None:
            cur = torch.cuda.current_stream(self.dev)
            cs = torch.cuda.Stream(device=self.dev)              # captured on a side stream (the current one may be the legacy default)
            cs.wait_stream(cur)
            with torch.cuda.device(self.dev), torch.cuda.stream(cs):
                for op in net["ops"]:                            # warm-up outside the capture (module loading, smem attributes)
                    op()
            cs.synchronize()
            g = torch.cuda.CUDAGraph()
            with torch.cuda.device(self.dev), torch.cuda.graph(g, stream=cs):
                for op in net["ops"]:
                    op()
            cur.wait_stream(cs)
            net["graphs"][stem_in] = g
        g.replay()

    def launches(self):
        """Kernel launches of one features() call: the crop kernel + the graph's kernels."""
        return 1 + len(self._net(1)["ops"])

    def features(self, pixels, crops):
        """pixels: uint8 device tensor of BGR pixels; crops: (n, 4) int64 rows {byte offset of the crop's first pixel, row pitch in
        bytes, height, width} (as ReidExtractor.features).  Returns (n, 512) float32 device features (not normalised)."""
        n = int(crops.shape[0])
        if n == 0:
            return torch.zeros((0, FEATURE_DIM), dtype=torch.float32, device=self.dev)
        if pixels.dtype != torch.uint8 or pixels.device != self.dev:
            raise L.B2TError("OsnetExtractor.features: pixels must be a uint8 tensor on %s" % self.dev)
        cr = crops.to(self.dev, torch.int64).contiguous()
        if tuple(cr.shape) != (n, 4):
            raise L.B2TError("OsnetExtractor.features: crops must be (n, 4)")
        net = self._net(n)
        H, W = self.size
        with torch.cuda.device(self.dev):
            self._check(self.lib.b2t_osnet_crops(C.c_void_p(pixels.data_ptr()), C.c_void_p(cr.data_ptr()), n, H, W, C.c_void_p(net["x4"].data_ptr()),
                                                 self.code, self._stream()), "b2t_osnet_crops")
            self._run(net, "x4")
        self.last_net = net
        return net["feat"][:n]

    def features_from_frame(self, frame, tlbrs):
        """StrongSORT.get_feature (strongsort.py:66-89): frame (H, W, 3) uint8 BGR, tlbrs (n, 4); the crops are
        ``ori_img[int(y1):int(y2), int(x1):int(x2)]``.  A negative coordinate after int() (the slice would wrap to the far side of the
        frame) or an empty crop (cv2.resize raises) raise B2TError.  Returns (n, 512) float32 device features; (0, 512) for no boxes."""
        t = np.asarray(tlbrs, dtype=np.float64).reshape(-1, 4)
        if len(t) == 0:
            return torch.zeros((0, FEATURE_DIM), dtype=torch.float32, device=self.dev)
        f = frame if isinstance(frame, torch.Tensor) else torch.from_numpy(np.ascontiguousarray(frame))
        if f.dtype != torch.uint8 or f.dim() != 3 or int(f.shape[2]) != 3:
            raise L.B2TError("OsnetExtractor.features_from_frame: frame must be (H, W, 3) uint8")
        f = f.to(self.dev).contiguous()
        Hf, Wf = int(f.shape[0]), int(f.shape[1])
        if not np.isfinite(t).all():
            raise L.B2TError("OsnetExtractor: a box coordinate is not finite")
        t = np.trunc(t).astype(np.int64)                                        # list(map(int, tlbr))
        if (t < 0).any():
            raise L.B2TError("OsnetExtractor: a box has a negative coordinate after int() (the reference's slice would wrap; clip the boxes first)")
        x1, y1 = np.minimum(t[:, 0], Wf), np.minimum(t[:, 1], Hf)
        x2, y2 = np.minimum(t[:, 2], Wf), np.minimum(t[:, 3], Hf)
        if ((x2 - x1) < 1).any() or ((y2 - y1) < 1).any():
            raise L.B2TError("OsnetExtractor: a crop is empty (cv2.resize raises on it in the reference)")
        crops = torch.from_numpy(np.stack([(y1 * Wf + x1) * 3, np.full_like(x1, 3 * Wf), y2 - y1, x2 - x1], 1))
        return self.features(f, crops)

    def forward_nchw(self, x):
        """x: (n, 3, H, W) float32 CUDA tensor, already preprocessed (H x W = size) -> (n, 512) float32 device features."""
        if not isinstance(x, torch.Tensor) or x.dtype != torch.float32 or x.dim() != 4 or int(x.shape[1]) != 3 or x.device != self.dev:
            raise L.B2TError("OsnetExtractor.forward_nchw: expected a float32 (n, 3, H, W) tensor on %s" % self.dev)
        if tuple(x.shape[2:]) != self.size:
            raise L.B2TError("OsnetExtractor.forward_nchw: input is %d x %d, the extractor was built for %d x %d" % (x.shape[2], x.shape[3], *self.size))
        n = int(x.shape[0])
        if n == 0:
            return torch.zeros((0, FEATURE_DIM), dtype=torch.float32, device=self.dev)
        x = x.contiguous()
        net = self._net(n)
        H, W = self.size
        if "x16" not in net:                                      # b2t_image_nhwc16's layout (3 channels padded to 16), made on first use
            net["x16"] = torch.zeros((net["n"], H, W, 16), dtype=self.dtype, device=self.dev)
        with torch.cuda.device(self.dev):
            self._check(self.lib.b2t_image_nhwc16(C.c_void_p(x.data_ptr()), C.c_void_p(net["x16"].data_ptr()), n, H, W, self.code, self._stream()),
                        "b2t_image_nhwc16")
            self._run(net, "x16")
        self.last_net = net
        return net["feat"][:n]


class OsnetSegments:
    """StrongSORT's crops of S sequences in ONE OSNet pass at a fixed capacity of `cap` crops, with nothing in a step that depends on a
    host-side count (TrackingPipeline with a StrongSORT engine).  ``cut`` builds the crop list on the device from the NMS output with
    b2t_reid_crops_from_dets -- the rows with score > det_thresh, StrongSORT's strict test (strongsort.py:118), by passing the next
    float32 above it to that kernel's >= test; ``run`` cuts and runs the network over all `cap` rows (padding rows repeat a valid crop)
    and scatters the feature of crop j to row rowmap[j] of ``feats`` (S, dmax, 512), the tensor TrackEngine.step_device(feats=) takes.
    An OSNet feature does not depend on the other crops of the pass (eval-mode BatchNorm), so one pass serves every sequence."""

    def __init__(self, ext, n_seq, dmax, cap):
        if n_seq < 1 or dmax < 1 or cap < 1:
            raise L.B2TError("OsnetSegments: n_seq, dmax and cap must be >= 1 (got %d, %d, %d)" % (n_seq, dmax, cap))
        self.ext, self.S, self.dmax, self.cap = ext, int(n_seq), int(dmax), int(cap)
        dev = ext.dev
        with torch.cuda.device(dev):
            self.crops = torch.zeros((self.cap, 4), dtype=torch.int64, device=dev)
            self.offsets = torch.zeros(self.S + 1, dtype=torch.int32, device=dev)
            self.rowmap = torch.full((self.cap,), -1, dtype=torch.int32, device=dev)
            self.status = torch.zeros(self.S + 1, dtype=torch.int32, device=dev)
            self._rows = torch.zeros((self.S * self.dmax + 1, FEATURE_DIM), dtype=torch.float32, device=dev)   # last row: padding sink
            self.feats = self._rows[: self.S * self.dmax].view(self.S, self.dmax, FEATURE_DIM)

    def capture(self):
        """Builds the network at this capacity and captures its graph (synchronises the device): a pass over 1 x 1 crops."""
        crops = torch.tensor([[0, 3, 1, 1]], dtype=torch.int64, device=self.ext.dev).repeat(self.cap, 1)
        self.ext.features(torch.zeros(3, dtype=torch.uint8, device=self.ext.dev), crops)
        torch.cuda.synchronize(self.ext.dev)

    def cut(self, frames, dets, det_count, det_thresh):
        """On the current stream: frames (S, H, W, 3) uint8 device tensor, dets (S, dmax, 6) float32, det_count (S,) int32 (the
        detector's out / out_count); det_thresh: the tracker's conf_thresh."""
        if tuple(dets.shape) != (self.S, self.dmax, 6) or dets.dtype != torch.float32 or det_count.dtype != torch.int32 or tuple(det_count.shape) != (self.S,):
            raise L.B2TError("OsnetSegments.cut: dets must be float32 (%d, %d, 6) and det_count int32 (%d,)" % (self.S, self.dmax, self.S))
        if frames.dtype != torch.uint8 or frames.dim() != 4 or int(frames.shape[0]) != self.S or int(frames.shape[3]) != 3 or not frames.is_contiguous():
            raise L.B2TError("OsnetSegments.cut: frames must be a contiguous uint8 (%d, H, W, 3) tensor" % self.S)
        H, W = int(frames.shape[1]), int(frames.shape[2])
        strict = float(np.nextafter(np.float32(det_thresh), np.float32(np.inf)))
        rc = self.ext.lib.b2t_reid_crops_from_dets(dets.data_ptr(), det_count.data_ptr(), self.S, self.dmax, strict, H, W, self.cap,
                                                   self.crops.data_ptr(), self.offsets.data_ptr(), self.rowmap.data_ptr(),
                                                   self.status.data_ptr(), self.ext._stream())
        self.ext._check(rc, "b2t_reid_crops_from_dets")

    def run(self, frames):
        """On the current stream, while `frames` (the buffer ``cut`` saw) is still valid: crops + network + scatter to ``feats``."""
        f = self.ext.features(frames, self.crops)
        sink = self.S * self.dmax
        idx = torch.where(self.rowmap >= 0, self.rowmap, torch.full_like(self.rowmap, sink)).long()
        self._rows.index_copy_(0, idx, f)

    def raise_for_status(self, status):
        """status: the (S + 1,) status words read back -> B2TError naming the first refused condition and sequence."""
        for s in range(self.S):
            bits = int(status[s])
            if bits & L.REID_OVERFLOW:
                raise L.B2TError("OSNet: sequence %d: the crops of this step (%d in all sequences) exceed reid_cap = %d" % (s, int(status[self.S]), self.cap))
            if bits & L.REID_ZERO_SIZE:
                raise L.B2TError("OSNet: sequence %d: a detection with score > det_thresh gives an empty crop (cv2.resize raises on it in the reference)" % s)
            if bits & L.REID_NEGATIVE:
                raise L.B2TError("OSNet: sequence %d: a detection with score > det_thresh has a negative coordinate after int() (the reference's slice would wrap)" % s)
