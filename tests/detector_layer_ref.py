"""TEST INFRASTRUCTURE: checks every launch of a detector forward against a float64 restatement of the same op, each layer
from the stored 16-bit values it actually read -- not from the image -- so the bar stays strict, per element, at any weights and
any size, even where the network is chaotic (a 1e-4 perturbation grows ~30x over the w6 layers).  A stale read, a wrong tap or
a misplaced concat slice shows up in exactly the layer where it happens.

The harness walks the ORACLE's layer list (``w6_layers()`` / ``tiny_layers()``), not the detector's plan.  It reads a chain of
stored outputs through ``get(key)`` (NCHW tensors, full batch):
    i                      output of layer i (concat: in the reference's channel order, e.g. tiny's SP concat as [m13|m9|m5|x])
    ("spp", i, name)       SPPCSPC temporaries: t1 (cv1), t2 (cv3), x1 (cv4), m5 / m9 / m13, t5 (cv5), y1 (cv6), y2 (cv2)
    ("raw", lvl)           Detect conv output of level lvl, fp32 (B, 3 * 85, h, w)
``detector_views`` maps a ``DetectorW6`` onto these keys; ``oracle_chain`` builds them from ``oracle.detector.forward``.

Bars:
* exact ops -- ReOrg / the tiny input conversion (from the fp32 image rounded once), upsample, the SPP / SP pools, MP, every concat:
  ``torch.equal`` with the float64 result;
* conv + bias + activation (each half of a stacked ELAN pair and the seven SPPCSPC convs included):  ref = act(conv64(x, w16) + b32)
  in float64, and per element
      |got - ref| <= 1/2 ulp16(|ref| + E) + E
      E = s_act * ((2 * ceil(K / 16) + splits) * 2^-23 * sum|w x| + |b| * 2^-24) + e_act
  fp32 accumulation with at most two roundings, possibly truncating, per k16 wgmma step (ceil(K / 16) steps of K = 16-padded Cin x k x k;
  the row-packed stem pads each kernel row to four pixels: 12 steps), one more per split-K partial sum and one for the bias add
  (the ``splits`` term covers |acc| * 2^-24); s_act = 1.1 bounds SiLU's slope (max 1.0998), 1 for LeakyReLU / identity;
  e_act = 1e-5 is the documented error of the one-tanh.approx SiLU epilogue, 0 otherwise (LeakyReLU's v * 0.1f rounding is
  covered: E >= 2^-22 |v| >= 2^-22 * 10 |out| there); sum|w x| is a second float64 conv of |x| and |w|;
* Detect heads (fp32, linear): |got - ref| <= E + ulp32(|ref| + E);
* decode: ``pred`` against a float64 decode of the stored fp32 ``raw`` with the bound of b2t_decode.cuh's fp32 formula (below);
* every value read must be finite: an inf or NaN (e.g. a tile left at a NaN sentinel) fails its layer.
These constants come from the arithmetic.  They are not fitted to a run.
"""
import math
from dataclasses import dataclass, field

import torch
import torch.nn.functional as F

_FMT = {torch.float16: (10, -14), torch.bfloat16: (7, -126), torch.float32: (23, -126)}     # (mantissa bits, min normal exponent)
NO = 85


def ulp(a, dtype):
    """ulp of the format `dtype` at float64 magnitudes a >= 0 (subnormal spacing below the smallest normal)."""
    p, emin = _FMT[dtype]
    _, e = torch.frexp(a)
    e = torch.where(a < 2.0 ** emin, torch.full_like(e, emin), e - 1)
    return torch.exp2((e - p).to(torch.float64))


def round_nearest(r, dtype):
    """float64 -> the nearest value of `dtype` (ties to even), computed in float64 (no double rounding through fp32)."""
    q = ulp(r.abs(), dtype)
    return torch.round(r / q) * q


def _resolve(i, f):
    return f if f >= 0 else i + f


@dataclass
class Row:
    key: object
    name: str
    kind: str                      # exact | conv | head | decode
    n: int = 0
    nonfinite: int = 0
    max_ratio: float = 0.0         # largest |err| / bound (exact ops: 0 if equal, inf otherwise)
    n_exact: int = 0               # elements equal to the correctly rounded float64 value
    ulp_sum: float = 0.0           # sum of sign(ref) * err / ulp(|ref|)
    note: str = ""
    images: list = field(default_factory=list)

    @property
    def ok(self):
        return self.nonfinite == 0 and self.max_ratio <= 1.0

    @property
    def frac_exact(self):
        return self.n_exact / max(self.n, 1)

    @property
    def mean_ulp(self):
        return self.ulp_sum / max(self.n, 1)


def _act64(v, act):
    if act == "silu":
        return v * torch.sigmoid(v)
    if act == "leaky":
        return torch.where(v >= 0, v, 0.1 * v)
    return v


def _ksteps(cin, k):
    if k == 3 and cin <= 16:
        return 12
    return (cin + 15) // 16 * k * k


def conv_reference(x, w16, b, k, s, act, out_dtype, splits=1):
    """float64 (ref, bound) of one conv launch: x float64 (the stored 16-bit values), w16 float64 (the weight rounded to the
    activation type), b fp32 bias as float64.  out_dtype: the stored type (fp32 = Detect head)."""
    pad = k // 2
    acc = F.conv2d(x, w16, None, stride=s, padding=pad)
    mag = F.conv2d(x.abs(), w16.abs(), None, stride=s, padding=pad)
    v = acc + b.view(1, -1, 1, 1)
    ref = _act64(v, act)
    s_act = 1.1 if act == "silu" else 1.0
    e_act = 1e-5 if act == "silu" else 0.0
    E = s_act * ((2 * math.ceil(_ksteps(w16.shape[1], k)) + splits) * 2.0 ** -23 * mag + b.abs().view(1, -1, 1, 1) * 2.0 ** -24) + e_act
    if out_dtype == torch.float32:
        bound = E + ulp(ref.abs() + E, torch.float32)
    else:
        bound = 0.5 * ulp(ref.abs() + E, out_dtype) + E
    return ref, bound


def decode_reference(raw, anchors, stride):
    """raw (1, 3 * 85, h, w) fp32 values as float64 -> (pred rows (1, 3 h w, 85), bound) for b2t_decode.cuh:
        s = 1 / (1 + expf(-r))                 expf within 2 ulp (CUDA C Programming Guide), + and / correctly rounded:
                                               |ds| <= s * (2^-22 + 2^-23) * (1 + 2^-20)
        xy = (s * 2 - 0.5 + g) * stride        two roundings (stride is a power of two): stride * (2 |ds| + 2^-24 (|2s - .5| + |2s - .5 + g|)) * (1 + 2^-20)
        wh = (s * 2) * (s * 2) * anchor        two roundings: |wh| * (2 |ds| / s + 2^-23) * (1 + 2^-20)
    plus 2^-126 absolute (the fp32 subnormal range)."""
    _, c, h, w = raw.shape
    r = raw.reshape(3, NO, h, w).permute(0, 2, 3, 1)                       # (a, y, x, o)
    s = 1.0 / (1.0 + torch.exp(-r))
    ds = s * (2.0 ** -22 + 2.0 ** -23)
    gy, gx = torch.meshgrid(torch.arange(h, device=raw.device, dtype=torch.float64), torch.arange(w, device=raw.device, dtype=torch.float64), indexing="ij")
    out, bound = s.clone(), ds.clone()
    for o, g in ((0, gx), (1, gy)):
        t = 2 * s[..., o] - 0.5
        out[..., o] = (t + g) * stride
        bound[..., o] = stride * (2 * ds[..., o] + 2.0 ** -24 * (t.abs() + (t + g).abs()))
    an = torch.tensor(anchors, dtype=torch.float64, device=raw.device).view(3, 2)
    for o in (2, 3):
        out[..., o] = (2 * s[..., o]) ** 2 * an[:, o - 2].view(3, 1, 1)
        bound[..., o] = out[..., o] * (2 * ds[..., o] / s[..., o] + 2.0 ** -23)
    return out.reshape(1, -1, NO), (bound * (1 + 2.0 ** -20) + 2.0 ** -126).reshape(1, -1, NO)


class _Image:
    """float64 copies of one image's stored tensors, made on first use."""

    def __init__(self, get, b, dev):
        self.get, self.b, self.dev, self.cache = get, b, dev, {}

    def __call__(self, key):
        if key not in self.cache:
            self.cache[key] = self.get(key)[self.b:self.b + 1].to(self.dev, torch.float64)
        return self.cache[key]


def check_chain(layers, sd, act, dtype, img, get, anchors, strides, images=None, name_offset=0, splits=1, pred=None, device=None):
    """Every layer of `layers` checked from the stored outputs `get` reads (see the module docstring) -> [Row], in layer order.
    img: the fp32 image batch the chain ran on; images: which batch entries to check (default all); pred: the decoded (B, N, 85)
    to check against the stored raw maps (optional); device: where the float64 reference runs (default: the image's)."""
    dev = device or img.device
    images = list(range(img.shape[0])) if images is None else list(images)
    rows = {}
    order = []

    def row(key, name, kind):
        if key not in rows:
            rows[key] = Row(key, name, kind)
            order.append(key)
        return rows[key]

    def weight(name):
        return sd[name + ".weight"].to(dev, torch.float32).to(dtype).double(), sd[name + ".bias"].to(dev, torch.float32).double()

    def finite(r, got):
        bad = int((~torch.isfinite(got)).sum())
        r.nonfinite += bad
        return bad == 0

    def exact(key, name, got, ref):
        r = row(key, name, "exact")
        r.n += got.numel()
        if not finite(r, got):
            return
        if ref.shape[1] < got.shape[1]:                                 # channel padding of the stem / input buffer: zeros
            ref = F.pad(ref, (0, 0, 0, 0, 0, got.shape[1] - ref.shape[1]))
        eq = got == ref
        r.n_exact += int(eq.sum())
        if got.shape != ref.shape or not torch.equal(got, ref):
            r.max_ratio = math.inf

    def conv(key, name, x, wname, k, s, got, out_dtype=None, act_=None):
        out_dtype = out_dtype or dtype
        r = row(key, name, "head" if out_dtype == torch.float32 else "conv")
        r.n += got.numel()
        w, b = weight(wname)
        x = x[:, :w.shape[1]]                                           # the stem / input buffer's zero padding channels
        if not (finite(r, got) & finite(r, x)):                         # a non-finite input fails its producer and every consumer
            return
        ref, bound = conv_reference(x, w, b, k, s, act if act_ is None else act_, out_dtype, splits)
        if got.shape != ref.shape:
            r.max_ratio, r.note = math.inf, "shape %s != %s" % (tuple(got.shape), tuple(ref.shape))
            return
        err = got - ref
        r.max_ratio = max(r.max_ratio, float((err.abs() / bound).max()))
        r.n_exact += int((got == round_nearest(ref, out_dtype)).sum())
        r.ulp_sum += float((err * torch.sign(ref) / ulp(ref.abs(), out_dtype)).sum())

    for b in images:
        X = _Image(get, b, dev)
        rimg = img[b:b + 1].to(dev, torch.float32).to(dtype).double()      # the fp32 image rounded once to the 16-bit type

        def inp(j):
            """the tensor a consumer of layer j reads: concats are assembled from their sources, in the reference's order"""
            if layers[j][1] == "concat":
                return torch.cat([inp(_resolve(j, f)) for f in layers[j][2]], 1)
            return X(j)

        for i, op, frm, args in layers:
            mi = i + name_offset
            if op == "reorg":
                ref = torch.cat([rimg[..., ::2, ::2], rimg[..., 1::2, ::2], rimg[..., ::2, 1::2], rimg[..., 1::2, 1::2]], 1)
                exact(i, "%d reorg" % i, X(i), ref)
            elif op == "input":
                exact(i, "%d input" % i, X(i), rimg)
            elif op == "mp":
                exact(i, "%d mp" % i, X(i), F.max_pool2d(inp(_resolve(i, frm)), 2, 2))
            elif op == "sp":
                exact(i, "%d sp%d" % (i, args[0]), X(i), F.max_pool2d(inp(_resolve(i, frm)), args[0], 1, args[0] // 2))
            elif op == "up":
                exact(i, "%d up" % i, X(i), F.interpolate(inp(_resolve(i, frm)), scale_factor=2, mode="nearest"))
            elif op == "concat":
                exact(i, "%d concat" % i, X(i), inp(i))
            elif op == "conv":
                conv(i, "%d conv%dx%d/%d" % (i, args[1], args[1], args[2]), inp(_resolve(i, frm)), "model.%d.conv" % mi, args[1], args[2], X(i))
            elif op == "sppcspc":
                p = "model.%d." % mi
                S = lambda nm: X(("spp", i, nm))                                      # noqa: E731
                xin = inp(_resolve(i, frm))
                conv(("spp", i, "t1"), "%d.cv1" % i, xin, p + "cv1.conv", 1, 1, S("t1"))
                conv(("spp", i, "t2"), "%d.cv3" % i, S("t1"), p + "cv3.conv", 3, 1, S("t2"))
                conv(("spp", i, "x1"), "%d.cv4" % i, S("t2"), p + "cv4.conv", 1, 1, S("x1"))
                for kk in (5, 9, 13):
                    exact(("spp", i, "m%d" % kk), "%d.pool%d" % (i, kk), S("m%d" % kk), F.max_pool2d(S("x1"), kk, 1, kk // 2))
                cat4 = torch.cat([S("x1"), S("m5"), S("m9"), S("m13")], 1)
                conv(("spp", i, "t5"), "%d.cv5" % i, cat4, p + "cv5.conv", 1, 1, S("t5"))
                conv(("spp", i, "y1"), "%d.cv6" % i, S("t5"), p + "cv6.conv", 3, 1, S("y1"))
                conv(("spp", i, "y2"), "%d.cv2" % i, xin, p + "cv2.conv", 1, 1, S("y2"))
                conv(i, "%d.cv7" % i, torch.cat([S("y1"), S("y2")], 1), p + "cv7.conv", 1, 1, X(i))
            elif op == "detect":
                off = 0
                for lvl, f in enumerate(frm):
                    raw = X(("raw", lvl))
                    conv(("raw", lvl), "%d.m.%d head" % (i, lvl), inp(f), "model.%d.m.%d" % (mi, lvl), 1, 1, raw, torch.float32, "linear")
                    if pred is not None:
                        r = row(("decode", lvl), "decode %d" % lvl, "decode")
                        n = 3 * raw.shape[2] * raw.shape[3]
                        got = pred[b:b + 1, off:off + n].to(dev, torch.float64)
                        r.n += got.numel()
                        if finite(r, got) & finite(r, raw):
                            ref, bound = decode_reference(raw, anchors[lvl], float(strides[lvl]))
                            r.max_ratio = max(r.max_ratio, float(((got - ref).abs() / bound).max()))
                            r.n_exact += int((got == round_nearest(ref, torch.float32)).sum())
                        off += n
        for r in rows.values():
            r.images.append(b)
    return [rows[k] for k in order]


def failures(rows):
    return [r for r in rows if not r.ok]


def format_table(rows, title=""):
    lines = [title] if title else []
    lines.append("%-22s %-6s %12s %10s %9s %11s %9s" % ("layer", "kind", "elements", "err/bound", "exact", "mean ulp", "nonfinite"))
    for r in rows:
        lines.append("%-22s %-6s %12d %10.3g %8.2f%% %+11.4f %9d%s" % (r.name, r.kind, r.n, r.max_ratio, 100 * r.frac_exact, r.mean_ulp, r.nonfinite,
                                                                       ("  " + r.note) if r.note else ("" if r.ok else "  FAIL")))
    return "\n".join(lines)


# ---------------------------------------------------------------- adapters

def _nchw(t):
    return t.permute(0, 3, 1, 2)


def detector_spans(det, layers):
    """key -> (NHWC buffer, first channel, channel count) of everything ``check_chain`` reads on a ``DetectorW6``; the ReOrg stem
    entry is the unpadded window of its row-padded buffer (see ``detector_views``)."""
    spans = {}
    for i, op, frm, args in layers:
        if op == "detect":
            for lvl in range(len(frm)):
                spans[("raw", lvl)] = (det.raw[lvl], 0, 3 * NO)
            continue
        buf, off = det.place[i]
        spans[i] = (buf, off, det.ch[i])
        if op == "sppcspc":
            t, c_ = det.spp_tmp[i], args[0]
            spans.update({("spp", i, "t1"): (t["t1"], 0, c_), ("spp", i, "t2"): (t["t2"], 0, c_), ("spp", i, "t5"): (t["t5"], 0, c_),
                          ("spp", i, "x1"): (t["cat4"], 0, c_), ("spp", i, "m5"): (t["cat4"], c_, c_), ("spp", i, "m9"): (t["cat4"], 2 * c_, c_),
                          ("spp", i, "m13"): (t["cat4"], 3 * c_, c_), ("spp", i, "y1"): (t["cat2"], 0, c_), ("spp", i, "y2"): (t["cat2"], c_, c_)})
    return spans


def detector_views(det, layers):
    """key -> NCHW view on the detector's buffers (no copies, except the tiny SP concat, which is gathered into the reference's order
    through ``det.in_perm``).  Layer 0: the ReOrg stem's unpadded window (one zero pixel on the left of every row) or the tiny
    input buffer, all 16 channels (the padding channels must hold zeros)."""
    views = {}
    for key, (buf, off, c) in detector_spans(det, layers).items():
        if key == 0 and det.stem_padded:
            views[key] = _nchw(buf[:, :, 1:1 + det.W // 2, :])
        elif isinstance(key, int) and key in det.in_perm:
            views[key] = _nchw(buf)[:, det.in_perm[key].to(buf.device)]
        else:
            views[key] = _nchw(buf[..., off:off + c])
    return views


def oracle_chain(layers, sd, img, anchors, strides, dtype, act="silu", name_offset=0):
    """The oracle's forward with the 16-bit rounding emulated, stored as the detector stores it (16-bit layers, fp32 heads):
    (store {key: tensor}, pred)."""
    from oracle import detector as OD
    with torch.no_grad():
        res = OD.forward(layers, sd, img, anchors, strides, emulate_bf16=dtype, act=act, name_offset=name_offset, return_layers=True)
    store = {}
    for i, t in enumerate(res["layers"]):
        if t is not None:
            store[i] = t.to(dtype)
    for i, d in res["spp"].items():
        for nm, t in d.items():
            store[("spp", i, nm)] = t.to(dtype)
    for lvl, t in enumerate(res["raw"]):
        store[("raw", lvl)] = t
    return store, res["pred"]
