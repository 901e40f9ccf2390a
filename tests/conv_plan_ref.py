"""TEST INFRASTRUCTURE: one conv launch as it is stored -- an NHWC channel slice of a possibly wider buffer, read from a slice of
another (or of the row-padded stem buffer) -- checked against the float64 bound of ``detector_layer_ref.conv_reference``, plus
the buffer around the slice: every element outside the slice must still hold the sentinel the buffer was filled with.

The one allowance outside the slice is the TMA store granule: a store clips at 16 bytes, so a slice whose channel count is not a
multiple of 8 (16-bit) / 4 (fp32) owns the channels up to the next granule (the 255-channel head owns channel 255 of its 256-wide
buffer); those are not checked.
"""
import math
from dataclasses import dataclass

import torch

import detector_layer_ref as R

ACT = {0: "linear", 1: "silu", 3: "leaky"}          # b2t_conv_desc.act -> the activation conv_reference applies


def unpack_weight(w_packed, cout, cin, k):
    """``pack_conv_weight``'s (Cout_rows, k * k * Cin) rows back to (Cout, Cin, k, k), in the packed (16-bit) type."""
    return w_packed[:cout].view(cout, k, k, cin).permute(0, 3, 1, 2)


def input_nchw(x, in_coff, cin, w, x_pixel0=0):
    """float64 NCHW copy of what a plan reads: channels [in_coff, in_coff + cin) of pixels [x_pixel0, x_pixel0 + w) of every row of
    the NHWC buffer x (rows may be wider than w: the padded ReOrg stem buffer)."""
    return x[:, :, x_pixel0:x_pixel0 + w, in_coff:in_coff + cin].permute(0, 3, 1, 2).double()


def granule_end(out_coff, cout, f32):
    gran = 4 if f32 else 8
    return out_coff + (cout + gran - 1) // gran * gran


class ConvRef:
    """float64 reference of one conv launch: x NCHW float64 (the stored 16-bit input values), w (Cout, Cin, k, k) in the 16-bit type
    (or its float64 values), b fp32 bias.  ``bound(splits)`` caches one (ref, bound) per split-K count."""

    def __init__(self, x, w, b, k, s, act, io_dtype, f32):
        self.x, self.w, self.b = x, w.double(), b.double()
        self.k, self.s, self.act = k, s, ACT[int(act)]
        self.out_dtype = torch.float32 if f32 else io_dtype
        self.f32 = bool(f32)
        self._cache = {}

    def __call__(self, splits=1):
        if splits not in self._cache:
            self._cache[splits] = R.conv_reference(self.x, self.w, self.b, self.k, self.s, self.act, self.out_dtype, splits)
        return self._cache[splits]


@dataclass
class Check:
    n: int                         # elements of the slice
    nonfinite: int                 # of them not finite (a tile left at a NaN sentinel)
    max_ratio: float               # largest |err| / bound over the finite ones
    n_exact: int                   # equal to the correctly rounded float64 value
    over: torch.Tensor             # (N, C, Ho, Wo) bool: over the bound or not finite
    outside: torch.Tensor          # (N, Ho, Wo, pitch) bool: outside the slice and its granule tail, no longer the sentinel

    @property
    def ok(self):
        return self.nonfinite == 0 and self.max_ratio <= 1.0 and not bool(self.outside.any())

    def where(self):
        """a short description of the first failing elements (NCHW indices of the slice, NHWC indices outside it)"""
        parts = []
        if bool(self.over.any()):
            idx = self.over.nonzero()
            parts.append("%d elements over the bound / not finite, first (n, c, y, x) %s" % (idx.shape[0], idx[:3].tolist()))
        if bool(self.outside.any()):
            idx = self.outside.nonzero()
            parts.append("%d elements outside the slice overwritten, first (n, y, x, channel) %s" % (idx.shape[0], idx[:3].tolist()))
        return "; ".join(parts) or "ok"


def sentinel_kept(t, sentinel):
    return torch.isnan(t) if isinstance(sentinel, float) and math.isnan(sentinel) else t == sentinel


def check_output(y, out_coff, cout, ref, bound, out_dtype, sentinel=float("nan")):
    """y: the NHWC output buffer after the launch; (ref, bound) from ``ConvRef``; sentinel: what y held before it."""
    f32 = out_dtype == torch.float32
    got = y[..., out_coff:out_coff + cout].permute(0, 3, 1, 2).to(ref.device, torch.float64)
    fin = torch.isfinite(got)
    ratio = torch.where(fin, (got - ref).abs() / bound, torch.zeros_like(got))
    over = ~fin | (ratio > 1.0)
    keep = torch.ones(y.shape[-1], dtype=torch.bool, device=y.device)
    keep[out_coff:granule_end(out_coff, cout, f32)] = False
    outside = keep.view(1, 1, 1, -1) & ~sentinel_kept(y, sentinel)
    return Check(n=got.numel(), nonfinite=int((~fin).sum()), max_ratio=float(ratio.max()) if got.numel() else 0.0,
                 n_exact=int((got == R.round_nearest(ref, out_dtype)).sum()), over=over, outside=outside)
