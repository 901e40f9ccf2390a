"""YOLOv7-w6 forward + decode + NMS on the H100 kernels (csrc/b2t_conv.cu, csrc/b2t_detect.cu).

Replaces, for the reference's detector boundary (SURVEY.md section 8b B-det):
  ``model(img)[0]``                     models/yolo.py:321-351 (forward_once) + :39-57 (Detect)
  ``non_max_suppression(...)``          utils/general.py:607-695
  ``scale_coords(...).round()``         utils/general.py:319-340, tracker/track.py:240

Activations are NHWC bf16 with fp32 accumulation in registers; the Detect logits stay fp32.  Every tensor that feeds a
``Concat`` is produced at its channel offset inside the concat buffer (no copies); the whole forward is a fixed
sequence of ~115 launches, optionally replayed as one CUDA graph.  ``detect()`` never materialises the (B, N, 85)
prediction tensor: the decode is fused into the NMS candidate filter; ``forward()`` / ``decode()`` produce it on request.
"""
import ctypes as C

import torch

from . import _lib as L
from .conv import ConvPlan, pack_conv_weight, pack_conv_weight_rowpack
from .w6 import ANCHORS, NO, STRIDES, layer_channels, stackable_pairs, w6_layers, _resolve


def _check(lib, rc, what):
    if rc != 0:
        raise L.B2TError("%s: %s" % (what, (lib.b2t_detect_last_error() or b"").decode()))


_TUNE_CACHE = {}      # layer signature -> (variant index, tile configuration, record): see DetectorW6._tuned_plan


class ConvVariants(list):
    """What ``conv_variants`` returns: the list of variants, plus ``out_geom`` = (n, ho, wo), the output map of the launch (None
    when it reads the padded stem buffer), from which ``conv_candidates`` decides whether pixel runs are worth timing."""
    def __init__(self, items, out_geom=None):
        super().__init__(items)
        self.out_geom = out_geom


def conv_variants(w, k, s, cin, dtype, stem_row=None, out_geom=None):
    """The addressing variants of one conv launch: [(packed weights, extra ConvPlan arguments)], the default first.  w: the fp32
    (Cout, Cin, k, k) weight, Cin already padded; stem_row: the row pitch in pixels when the conv reads the padded ReOrg stem buffer;
    out_geom: (n, ho, wo) of the output map."""
    if stem_row is not None:        # the stem reads the padded ReOrg buffer: row-packed first, generic addressing as the fallback
        return ConvVariants([(pack_conv_weight_rowpack(w, dtype=dtype), dict(rowpack=True, in_row_pixels=stem_row, x_pixel0=0)),
                             (pack_conv_weight(w, dtype=dtype), dict(in_row_pixels=stem_row, x_pixel0=1)),
                             (pack_conv_weight(w, dtype=dtype), dict(in_row_pixels=stem_row, x_pixel0=1, halo=1))])
    variants = ConvVariants([(pack_conv_weight(w, dtype=dtype), {})], out_geom)
    if k == 3 and s == 1 and cin % 64 == 0:         # halo-tile addressing competes with one-tile-per-tap
        variants.append((variants[0][0], dict(halo=1)))
    return variants


def pixel_runs_pay(k, out_geom):
    """True when a 3x3 layer's best spatial patch (TH x TW = 128 pixels, TW 4, 8 or 16) computes more pixel slots than runs of 128
    pixels of the flattened N*Ho*Wo axis (tile_w = 128) -- the 20 x 20 and 40 x 40 maps of w6 -- so exactly divisible maps pay
    no extra tuning time."""
    if k != 3 or out_geom is None:
        return False
    n, ho, wo = out_geom
    patch = min(-(-ho // (128 // tw)) * -(-wo // tw) for tw in (4, 8, 16)) * 128 * n
    return patch > -(-n * ho * wo // 128) * 128


def conv_candidates(k, s, cin, cout, f32, variants):
    """Every (variant index, tile configuration) the autotuner times for one conv launch, in timing order: tile width BLOCK_N, one or
    two 128-pixel sub-tiles per tile (mt), ring depth (0 = as deep as shared memory allows, 2 / 3 = shallow rings) and, for 1x1 layers
    with whole 128-channel pairs, one or two K chunks per ring stage (kpair), for each addressing variant.  BLOCK_N 32 is offered to
    layers of at most 32 channels only, where it is the kernel's default tiling.  Where ``pixel_runs_pay``, variant 0 is also offered
    as 128-pixel runs (tile_w = 128) with the same grid.  Some are refused by ``b2t_conv_plan_create`` for a given layer (B2TError);
    the autotuner skips those."""
    cout_pad = (cout + 15) // 16 * 16
    kpairs = (1, 2) if (k == 1 and s == 1 and cin % 128 == 0) else (0,)
    shapes = [dict(block_n=bn, mt=mt, stages=st, kpair=kp) for bn in (32, 64, 128, 256) for mt in (1, 2) for st in (0, 2, 3) for kp in kpairs
              if (bn >= 64 or cout_pad <= 32) and bn <= max(64, cout_pad) and 2 * mt * bn <= 512 and not (f32 and mt == 2 and bn > 64)]
    runs = [(0, dict(cfg, tile_w=128)) for cfg in shapes] if pixel_runs_pay(k, getattr(variants, "out_geom", None)) else []
    return [(vi, cfg) for vi in range(len(variants)) for cfg in shapes] + runs


class DetectorW6:
    def __init__(self, state_dict, batch=1, img_size=1280, device="cuda:0", conf_thres=0.01, iou_thres=0.45, max_det=300,
                 max_nms=30000, use_graph=True, autotune=True, fuse_pairs=True, act_dtype=torch.float16,
                 layers=None, anchors=ANCHORS, strides=STRIDES, act=1, total_stride=64, name_offset=0):
        """layers / anchors / strides / act: the graph (default: YOLOv7-w6, SiLU).  ``b200track.tiny.DetectorTiny`` passes the
        YOLOv7-tiny graph (LeakyReLU(0.1) = act 3, MP / SP pools, three Detect levels, total stride 32)."""
        if not torch.cuda.is_available():
            raise L.B2TError("DetectorW6 needs a CUDA device (H100, sm_90a); there is no CPU fallback")
        # img_size: int (square) or (height, width) -- e.g. the 768 x 1280 minimum rectangle a letterboxed 1080p frame becomes
        H, W = (img_size, img_size) if isinstance(img_size, int) else (int(img_size[0]), int(img_size[1]))
        assert H % total_stride == 0 and W % total_stride == 0, "image sides must be multiples of the graph's total stride (w6: 64 = ReOrg / 2 and five stride-2 convs)"
        self.conv_act, self.anchors, self.strides = act, anchors, strides
        no_ = name_offset              # layer index -> the reference's module index (the tiny graph has an explicit input op in front)
        self.lib = L.load()
        # 16-bit type of activations and weights: fp16 (default; the reference's own GPU half mode, detect.py:41) or bf16 --
        # the same wgmma rate, fp32 accumulation either way; fp16 keeps 3 more mantissa bits, bf16 the fp32 range
        self.act_dtype = act_dtype
        self.act_code = L.act_dtype_code(act_dtype)
        self.dev = torch.device(device)
        self.B, self.H, self.W = batch, H, W
        self.S = H if H == W else None
        self.conf_thres, self.iou_thres, self.max_det, self.max_nms = conf_thres, iou_thres, max_det, max_nms
        layers = layers if layers is not None else w6_layers()
        ch = layer_channels(layers)
        n = len(layers)
        # ---- spatial size (h, w) of every layer output
        hw = [(0, 0)] * n
        for i, op, frm, args in layers:
            if op == "reorg":
                hw[i] = (H // 2, W // 2)
            elif op == "input":
                hw[i] = (H, W)
            elif op == "mp":
                ph, pw = hw[_resolve(i, frm)]
                hw[i] = (ph // 2, pw // 2)
            elif op == "sp":
                hw[i] = hw[_resolve(i, frm)]
            elif op == "conv":
                ph, pw = hw[_resolve(i, frm)]
                hw[i] = (ph // args[2], pw // args[2])
            elif op == "concat":
                hw[i] = hw[_resolve(i, frm[0])]
            elif op == "up":
                ph, pw = hw[_resolve(i, frm)]
                hw[i] = (ph * 2, pw * 2)
            elif op == "sppcspc":
                hw[i] = hw[_resolve(i, frm)]
        self.hw, self.ch = hw, ch
        # ---- placement: tensors consumed by a concat live inside the concat buffer
        place = {}                      # tensor index -> (buffer, channel offset)
        bufs = {}

        def new_buf(hw_, c, dtype=act_dtype):
            return torch.zeros((batch, hw_[0], hw_[1], c), dtype=dtype, device=self.dev)

        self.in_perm = {}               # concat index -> our channel -> reference channel (when the buffer order differs from `frm`)
        for i, op, frm, args in layers:
            if op == "concat":
                buf = new_buf(hw[i], ch[i])
                bufs[i] = buf
                srcs = [_resolve(i, f) for f in frm]
                order = list(srcs)
                sp = [j for j in srcs if layers[j][1] == "sp"]
                if sp:
                    # YOLOv7-tiny's SPP: cat(SP13(x), SP9(x), SP5(x), x).  The pooling kernel writes [x | m5 | m9 | m13]: the buffer takes
                    # that order and the consuming conv gets its input channels permuted instead
                    x_src = _resolve(sp[0], layers[sp[0]][2])
                    assert len(sp) == 3 and sorted(srcs) == sorted(sp + [x_src]) and sorted(layers[j][3][0] for j in sp) == [5, 9, 13]
                    order = [x_src] + sorted(sp, key=lambda j: layers[j][3][0])
                    ref_off, o = {}, 0
                    for j in srcs:
                        ref_off[j] = o
                        o += ch[j]
                    self.in_perm[i] = torch.cat([torch.arange(ref_off[j], ref_off[j] + ch[j]) for j in order])
                off = 0
                for j in order:
                    assert j not in place, "tensor %d feeds two concats" % j
                    place[j] = (buf, off)
                    off += ch[j]
                place[i] = (buf, 0)
        ch[0] = 16                      # ReOrg output / the image are padded to 16 channels for the tensor-core K granularity
        self.stem_padded = layers[0][1] == "reorg"
        if self.stem_padded:
            # ReOrg output rows carry one zero pixel on the left and zeros on the right (never written): the padded layout the
            # row-packed stem conv reads (b2t_conv_desc.rowpack)
            self.stem_row = hw[0][1] + 8
            place[0] = (torch.zeros((batch, hw[0][0], self.stem_row, 16), dtype=act_dtype, device=self.dev), 0)
        else:
            self.stem_row = hw[0][1]
            place[0] = (new_buf(hw[0], 16), 0)
        for i, op, frm, args in layers:
            if op in ("conv", "up", "sppcspc", "mp") and i not in place:
                place[i] = (new_buf(hw[i], ch[i]), 0)
        self.place = place
        self.autotune, self.tuned = autotune, {}
        # one read-only record per conv launch, for per-launch checks: source / destination buffers and channel offsets, every
        # addressing variant the autotuner offers for it (packed weights, extra ConvPlan arguments), the bias, the geometry, and the
        # (variant index, tile configuration) this detector runs
        self.conv_specs = []
        self.ops = []                   # (callable, flops)
        self.keep = []
        sd = state_dict

        def conv_op(name, src, cin, dst, cout, k, s, hw_in, act=None, f32=False, in_perm=None):
            act = self.conv_act if act is None else act
            names = name if isinstance(name, (list, tuple)) else [name]      # several convs of the SAME input = one conv with stacked rows
            w = torch.cat([sd[nm + ".weight"].to(self.dev, torch.float32) for nm in names], 0)
            if in_perm is not None:
                w = w[:, in_perm.to(self.dev)].contiguous()
            cin_real = w.shape[1]                                          # algorithmic flops count the real 12 stem channels, not the padded 16
            if w.shape[1] != cin:      # stem: 12 -> 16 zero-padded input channels
                wp = torch.zeros((w.shape[0], cin, k, k), device=self.dev)
                wp[:, :w.shape[1]] = w
                w = wp
            b = torch.cat([sd[nm + ".bias"].to(self.dev, torch.float32) for nm in names], 0).contiguous()
            name = "+".join(names)
            assert w.shape[0] == cout
            stem = src[0] is place[0][0] and self.stem_padded
            out_geom = (self.B, (hw_in[0] + 2 * (k // 2) - k) // s + 1, (hw_in[1] + 2 * (k // 2) - k) // s + 1)
            variants = conv_variants(w, k, s, cin, act_dtype, self.stem_row if stem else None, out_geom)
            # untuned: the first variant the kernel accepts (the stem falls back from row-packed to generic addressing)
            plan, vi, cfg = self._tuned_plan(src, variants if (self.autotune or stem) else variants[:1], b, dst, hw_in, cin, cout, k, s, act, f32)
            self.conv_specs.append(dict(name=name, op=len(self.ops), src=src[0], in_coff=src[1], dst=dst[0], out_coff=dst[1], variants=variants, bias=b,
                                        hw_in=tuple(hw_in), cin=cin, cout=cout, k=k, s=s, act=int(act), f32=bool(f32), chosen=(vi, dict(cfg))))
            self.keep.append(plan)
            flops = 2.0 * self.B * (hw_in[0] // s) * (hw_in[1] // s) * cout * k * k * cin_real
            self.ops.append((plan.run, flops, name))

        lib = self.lib
        stream = lambda: C.c_void_p(torch.cuda.current_stream(self.dev).cuda_stream)  # noqa: E731
        self.raw, self.decode_ops = [], []
        self.spp_tmp = {}               # SPPCSPC layer index -> its temporaries: t1 (cv1), t2 (cv3), cat4 = [cv4 | m5 | m9 | m13], t5 (cv5), cat2 = [cv6 | cv2]
        levels = []
        fused_away = set()
        pairs = set(stackable_pairs(layers)) if fuse_pairs else set()
        for i, op, frm, args in layers:
            if op == "reorg":
                dst = place[i][0]
                self.ops.append((lambda dst=dst: _check(lib, lib.b2t_image_reorg_padded(C.c_void_p(self.img.data_ptr()), C.c_void_p(dst.data_ptr()),
                                                                                          batch, H, W, self.stem_row, 1, self.act_code, stream()),
                                                         "image_reorg"), 0.0, "reorg"))
            elif op == "input":
                dst = place[i][0]
                self.ops.append((lambda dst=dst: _check(lib, lib.b2t_image_nhwc16(C.c_void_p(self.img.data_ptr()), C.c_void_p(dst.data_ptr()), batch, H, W,
                                                                                   self.act_code, stream()), "image_nhwc16"), 0.0, "input"))
            elif op == "mp":
                j = _resolve(i, frm)
                (sb, so), (db, do) = place[j], place[i]
                assert so == 0 and do == 0 and sb.shape[-1] == ch[j] and db.shape[-1] == ch[j], "MP reads and writes whole buffers"
                self.ops.append((lambda sb=sb, db=db, h=hw[j][0], w=hw[j][1], c=ch[j]: _check(lib, lib.b2t_maxpool2x2s2(
                    C.c_void_p(sb.data_ptr()), C.c_void_p(db.data_ptr()), batch, h, w, c, self.act_code, stream()), "maxpool2x2s2"), 0.0, "mp%d" % i))
            elif op == "sp":
                if args[0] == 5:               # one launch computes the 5 / 9 / 13 pools into the three slices that follow x in the concat buffer
                    j = _resolve(i, frm)
                    (sb, so), c = place[j], ch[j]
                    assert so == 0 and place[i] == (sb, c), "SP pools follow their input inside the concat buffer"
                    self.ops.append((lambda sb=sb, c=c, h=hw[j]: _check(lib, lib.b2t_spp_pool(C.c_void_p(sb.data_ptr()), sb.shape[-1], c, batch, h[0], h[1],
                                                                                              self.act_code, stream()), "spp_pool"), 0.0, "spp_pool"))
            elif op == "conv":
                if i in fused_away:
                    continue
                j = _resolve(i, frm)
                # the two parallel 1x1 convs that open every ELAN block read the same tensor and write adjacent slices of the
                # block's concat buffer ([... | conv(-2) | conv(-1)]): one launch with the weight rows stacked reads the input once
                if (i, i + 1) in pairs:
                    assert place[i + 1][0] is place[i][0] and place[i + 1][1] + ch[i + 1] == place[i][1]
                    fused_away.add(i + 1)
                    conv_op(["model.%d.conv" % (i + 1 + no_), "model.%d.conv" % (i + no_)], place[j], ch[j], place[i + 1], ch[i + 1] + ch[i], 1, 1, hw[j])
                else:
                    conv_op("model.%d.conv" % (i + no_), place[j], ch[j], place[i], args[0], args[1], args[2], hw[j], in_perm=self.in_perm.get(j))
            elif op == "up":
                j = _resolve(i, frm)
                (sb, so), (db, do) = place[j], place[i]
                self.ops.append((lambda sb=sb, so=so, db=db, do=do, h=hw[j][0], w=hw[j][1], c=ch[j]: _check(lib, lib.b2t_upsample2x(
                    C.c_void_p(sb.data_ptr()), sb.shape[-1], so, C.c_void_p(db.data_ptr()), db.shape[-1], do, batch, h, w, c, stream()),
                    "upsample2x"), 0.0, "up%d" % i))
            elif op == "sppcspc":
                j = _resolve(i, frm)
                c1, c2, h = ch[j], args[0], hw[j]
                c_ = c2
                t1, t2 = new_buf(h, c_), new_buf(h, c_)
                cat4, t5, cat2 = new_buf(h, 4 * c_), new_buf(h, c_), new_buf(h, 2 * c_)
                self.spp_tmp[i] = dict(t1=t1, t2=t2, cat4=cat4, t5=t5, cat2=cat2)      # read-only record, for per-layer checks
                pre = "model.%d." % (i + no_)
                conv_op(pre + "cv1.conv", place[j], c1, (t1, 0), c_, 1, 1, h)
                conv_op(pre + "cv3.conv", (t1, 0), c_, (t2, 0), c_, 3, 1, h)
                conv_op(pre + "cv4.conv", (t2, 0), c_, (cat4, 0), c_, 1, 1, h)
                self.ops.append((lambda cat4=cat4, c_=c_, h=h: _check(lib, lib.b2t_spp_pool(C.c_void_p(cat4.data_ptr()), cat4.shape[-1], c_, batch, h[0], h[1],
                                                                                              self.act_code, stream()), "spp_pool"), 0.0, "spp_pool"))
                conv_op(pre + "cv5.conv", (cat4, 0), 4 * c_, (t5, 0), c_, 1, 1, h)
                conv_op(pre + "cv6.conv", (t5, 0), c_, (cat2, 0), c_, 3, 1, h)
                conv_op(pre + "cv2.conv", place[j], c1, (cat2, c_), c_, 1, 1, h)
                conv_op(pre + "cv7.conv", (cat2, 0), 2 * c_, place[i], c2, 1, 1, h)
            elif op == "detect":
                self.n_total = sum(3 * hw[f][0] * hw[f][1] for f in frm)
                self.pred = torch.zeros((batch, self.n_total, NO), dtype=torch.float32, device=self.dev)
                off = 0
                for lvl, f in enumerate(frm):
                    raw = new_buf(hw[f], 256, torch.float32)
                    self.raw.append(raw)
                    conv_op("model.%d.m.%d" % (i + no_, lvl), place[f], ch[f], (raw, 0), 3 * NO, 1, 1, hw[f], act=False, f32=True)
                    anc = (C.c_float * 6)(*[float(v) for v in anchors[lvl]])
                    self.keep.append(anc)
                    self.decode_ops.append((lambda raw=raw, h=hw[f][0], w=hw[f][1], off=off, st=float(strides[lvl]), anc=anc: _check(lib, lib.b2t_detect_decode(
                        C.c_void_p(raw.data_ptr()), 256, C.c_void_p(self.pred.data_ptr()), batch, h, w, 3, NO, off, self.n_total, st, anc, stream()),
                        "detect_decode"), 0.0, "decode%d" % lvl))
                    levels.append((raw, hw[f], float(strides[lvl]), [float(v) for v in anchors[lvl]], off))
                    off += 3 * hw[f][0] * hw[f][1]
        self.head_levels = (L.HeadLevel * len(levels))()
        for k, (raw, (h, w), st, anc, off) in enumerate(levels):
            hl = self.head_levels[k]
            hl.raw, hl.raw_pitch, hl.h, hl.w, hl.stride, hl.level_off = raw.data_ptr(), 256, h, w, st, off
            for j in range(6):
                hl.anchors[j] = anc[j]
        self.flops = sum(f for _, f, _ in self.ops)
        self.img = torch.zeros((batch, 3, H, W), dtype=torch.float32, device=self.dev)
        self.out = torch.zeros((batch, max_det, 6), dtype=torch.float32, device=self.dev)
        self.out_count = torch.zeros(batch, dtype=torch.int32, device=self.dev)
        self.max_cand = self.n_total
        ws = lib.b2t_nms_workspace_bytes(batch, self.max_cand, max_nms)
        self.nms_ws = torch.empty(ws, dtype=torch.uint8, device=self.dev)
        # post-processing geometry of the NMS output (gain, pad_w, pad_h, clip width, clip height): the identity on the canvas until
        # set_source_frames declares the frames' size, then scale_coords back to the source frame (tracker/track.py:240)
        self.post_geo = (1.0, 0.0, 0.0, float(W), float(H))
        self.graph, self.graph_post = None, None
        self.fwd_graph = None
        self.use_graph = use_graph

    def _tuned_plan(self, src, variants, b, dst, hw_in, cin, cout, k, s, act, f32):
        """Plan-time autotuning: the kernel's best tiling depends on the layer -- tile width BLOCK_N, one or two 128-pixel
        sub-tiles per tile (mt), ring depth (0 = as deep as shared memory allows, 2 / 3 = shallow rings) and the addressing
        variant -- so each candidate of ``conv_candidates`` is timed with CUDA events on the real buffers and the fastest kept
        (tools/conv_layer_bench.py prints the whole table).  ``variants``: [(packed weights, extra ConvPlan arguments)].
        Returns (plan, variant index, tile configuration); untuned: the first variant accepted with the kernel's default tiling."""
        cands = conv_candidates(k, s, cin, cout, f32, variants) if self.autotune else [(vi, {}) for vi in range(len(variants))]
        # one tuning per process and layer signature: a second detector of the same shape (tests, the bench's arms) gets the SAME
        # plans without a second tuning pass.  (Every candidate sums each output in the same order -- csrc/b2t_conv.cu -- so the
        # choice changes the time, not the result.)
        key = (str(self.dev), self.B, tuple(hw_in), cin, cout, k, s, bool(act), bool(f32), str(src[0].dtype), src[0].shape[-1], src[1], dst[0].shape[-1], dst[1],
               tuple(tuple(sorted(e.items())) for _, e in variants))
        if self.autotune and key in _TUNE_CACHE:
            vi, cfg, rec = _TUNE_CACHE[key]
            self.tuned[len(self.ops)] = dict(rec)
            return (ConvPlan(src[0], variants[vi][0], b, dst[0], self.B, hw_in[0], hw_in[1], cin, src[1], cout, k, s, dst[1], act=act, out_f32=f32,
                             **cfg, **variants[vi][1]), vi, cfg)
        best, best_ms = None, None
        for vi, cfg in cands:
            wpk, extra = variants[vi]
            try:
                plan = ConvPlan(src[0], wpk, b, dst[0], self.B, hw_in[0], hw_in[1], cin, src[1], cout, k, s, dst[1], act=act, out_f32=f32,
                                **cfg, **extra)
            except L.B2TError:
                continue
            if not self.autotune:
                return plan, vi, cfg
            plan.run(); plan.run()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(4):
                plan.run()
            e1.record()
            torch.cuda.synchronize()
            ms = e0.elapsed_time(e1)
            if best_ms is None or ms < best_ms:
                best, best_ms = (plan, vi, dict(cfg)), ms
                self.tuned[len(self.ops)] = dict(cfg, variant=vi, us=ms * 250.0, **{k_: plan.info[k_] for k_ in ("grid", "stages", "smem")})
                _TUNE_CACHE[key] = (vi, dict(cfg), dict(self.tuned[len(self.ops)]))
        if best is None:
            raise L.B2TError("no valid conv configuration")
        return best

    # ---- pieces
    def _forward_launches(self):
        for fn, _, _ in self.ops:
            fn()

    def _nms_launch(self, post=True):
        """Detect decode fused with NMS, straight from the four raw head maps (b2t_detect_nms): `pred` is not touched.  post: rows
        scaled to the source frame declared by set_source_frames (the canvas when none was), clipped and rounded."""
        lib = self.lib
        rc = lib.b2t_detect_nms(C.cast(self.head_levels, C.c_void_p), len(self.head_levels), self.B, NO, self.conf_thres, self.iou_thres,
                                self.max_det, self.max_nms, self.max_cand, int(post), *self.post_geo,
                                C.c_void_p(self.nms_ws.data_ptr()), self.nms_ws.numel(), C.c_void_p(self.out.data_ptr()),
                                C.c_void_p(self.out_count.data_ptr()), C.c_void_p(torch.cuda.current_stream(self.dev).cuda_stream))
        _check(lib, rc, "detect_nms")

    def nms_from_pred(self, post=True):
        """non_max_suppression on the materialised `pred` tensor (b2t_nms) -- the two-step path decode() + NMS."""
        lib = self.lib
        rc = lib.b2t_nms(C.c_void_p(self.pred.data_ptr()), self.B, self.n_total, NO, self.conf_thres, self.iou_thres, self.max_det, self.max_nms,
                         self.max_cand, int(post), *self.post_geo, C.c_void_p(self.nms_ws.data_ptr()),
                         self.nms_ws.numel(), C.c_void_p(self.out.data_ptr()), C.c_void_p(self.out_count.data_ptr()),
                         C.c_void_p(torch.cuda.current_stream(self.dev).cuda_stream))
        _check(lib, rc, "nms")
        return self.out, self.out_count

    def decode(self):
        """Detect.forward's inference decode of the current raw head maps -> pred (B, N, 85) fp32 (what `model(img)[0]` is)."""
        for fn, _, _ in self.decode_ops:
            fn()
        return self.pred

    def set_source_frames(self, src_hw):
        """uint8 ingest: declare the (height, width) of the raw BGR frames this detector will be fed.  Allocates the device
        staging buffer ``self.src_u8`` (B, h, w, 3) and checks that the reference's letterbox geometry
        (tracker/tracker_dataloader.py:100-126, stride 64 minimum rectangle) produces exactly this detector's (H, W).
        From then on post-processed NMS rows (``detect(post=True)``, ``nms_from_pred(True)``, the pipeline) are in source-frame
        pixels: scale_coords from the canvas to (h, w), clipped to the frame, rounded (tracker/track.py:240)."""
        from .preprocess import letterbox_geometry, scale_coords_geometry
        if not self.stem_padded:
            raise L.B2TError("the uint8 ingest writes the ReOrg layout of the w6 stem: this graph takes the float tensor")
        h, w = int(src_hw[0]), int(src_hw[1])
        geo = letterbox_geometry((h, w), (max(self.H, self.W), max(self.H, self.W)), 64, True)
        if (geo["out_h"], geo["out_w"]) != (self.H, self.W):
            raise L.B2TError("frames of %dx%d letterbox to %dx%d, this detector was planned for %dx%d" % (h, w, geo["out_h"], geo["out_w"], self.H, self.W))
        self.src_geo, self.src_hw = geo, (h, w)
        post_geo = scale_coords_geometry((self.H, self.W), (h, w)) + (float(w), float(h))
        if post_geo != self.post_geo:
            self.graph = None                                                  # the captured NMS epilogue scales differently: capture again
        self.post_geo = post_geo
        self.src_u8 = torch.zeros((self.B, h, w, 3), dtype=torch.uint8, device=self.dev)
        return geo

    def ingest_u8_launch(self):
        """``self.src_u8`` (uint8 BGR frames, as cv2.imread returns them) -> letterbox + BGR->RGB + /255 + ReOrg + 16-bit NHWC straight
        into the stem's padded input buffer (b2t_letterbox_reorg): replaces ``self.ops[0]`` (ReOrg of the float tensor) when the
        frames arrive as bytes -- 3 bytes per pixel over PCIe instead of 12, and the float tensor never exists."""
        from .preprocess import launch_letterbox_reorg
        h, w = self.src_hw
        launch_letterbox_reorg(self.lib, self.src_u8.data_ptr(), self.B, h, w, 3 * w, self.src_geo, self.place[0][0].data_ptr(), self.stem_row, 1,
                               C.c_void_p(torch.cuda.current_stream(self.dev).cuda_stream), act_dtype=self.act_code)

    def forward(self, img=None):
        """img: (B,3,S,S) float32 in [0,1] on the device (or None to reuse self.img) -> pred (B, N, 85) fp32.
        With use_graph the ~105 launches (forward + decode) replay as one CUDA graph."""
        if img is not None:
            self.img.copy_(img, non_blocking=True)
        if self.use_graph:
            if self.fwd_graph is None:
                torch.cuda.synchronize()
                s = torch.cuda.Stream(device=self.dev)
                with torch.cuda.stream(s):
                    self._forward_launches(); self.decode()                    # warm-up outside capture
                    torch.cuda.synchronize()
                    self.fwd_graph = torch.cuda.CUDAGraph()
                    with torch.cuda.graph(self.fwd_graph, stream=s):
                        self._forward_launches()
                        self.decode()
                torch.cuda.synchronize()
            self.fwd_graph.replay()
            return self.pred
        self._forward_launches()
        return self.decode()

    def detect(self, img=None, post=True):
        """forward + NMS (+ scale_coords/clip/round): returns (out (B, max_det, 6), count (B,)) device tensors."""
        if img is not None:
            self.img.copy_(img, non_blocking=True)
        if self.use_graph:
            if self.graph is not None and self.graph_post != bool(post):
                self.graph = None                                              # the captured NMS epilogue differs: capture again
            if self.graph is None:
                self.graph_post = bool(post)
                torch.cuda.synchronize()
                s = torch.cuda.Stream(device=self.dev)
                with torch.cuda.stream(s):
                    self._forward_launches(); self._nms_launch(post)          # warm-up outside capture
                    torch.cuda.synchronize()
                    self.graph = torch.cuda.CUDAGraph()
                    with torch.cuda.graph(self.graph, stream=s):
                        self._forward_launches()
                        self._nms_launch(post)
                torch.cuda.synchronize()
            self.graph.replay()
        else:
            self._forward_launches()
            self._nms_launch(post)
        return self.out, self.out_count
