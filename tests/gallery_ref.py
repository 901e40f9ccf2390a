"""Checker for the gallery appearance cost (csrc/b2t_gallery.cu, DeepSORT's matching.nearest_embedding_distance).

  bound(feat_dim)      the kernel's derived error bound against the exact float64 value (restated from the kernel's header comment)
  pack(x)              NumPy restatement of b2t_gallery_pack: v = 2^8 x / |x| in float64, hi = fp16(v), lo = fp16(v - hi)
  exact(gal, counts, dets)   min over each slot's first counts[t] rows of 1 - u_g . u_f, u = x / |x| in float64 (+inf for no rows)
  reference_normalised(x)    the reference's cal_cosine_distance rows: x / np.linalg.norm(x) in float32
  adversarial_rows(rng, n, d)  mixed magnitudes (hi and lo in the fp16 subnormal range), large norms, a dominant element
"""
import math

import numpy as np

SCALE = 256.0


def bound(feat_dim):
    chunks = -(-feat_dim // 64)
    return (216 * 2.0 ** -23 + chunks * 2.0 ** -24) * (1 + 2.0 ** -9) + 3 * 2.0 ** -22 + 2.0 ** -32 * math.sqrt(feat_dim) + 2.0 ** -48


def unit(x):
    x = np.asarray(x, dtype=np.float64)
    return x / np.sqrt((x * x).sum(-1, keepdims=True))


def pack(x):
    v = unit(np.asarray(x, dtype=np.float32)) * SCALE
    hi = v.astype(np.float16)
    lo = (v - hi.astype(np.float64)).astype(np.float16)
    return hi, lo


def packed_dot(ga, gb):
    """the dot product the kernel forms, in float64 (no accumulation error): hi.hi + hi.lo + lo.hi over 2^16"""
    (ah, al), (bh, bl) = ga, gb
    ah, al, bh, bl = (t.astype(np.float64) for t in (ah, al, bh, bl))
    return (ah @ bh.T + ah @ bl.T + al @ bh.T) / SCALE ** 2


def exact(gal, counts, dets):
    gal = np.asarray(gal, dtype=np.float32)
    dets = np.asarray(dets, dtype=np.float32)
    out = np.full((gal.shape[0], dets.shape[0]), np.inf)
    ud = unit(dets)
    for t, c in enumerate(counts):
        c = max(0, min(int(c), gal.shape[1]))
        if c and len(dets):
            out[t] = (1.0 - unit(gal[t, :c]) @ ud.T).min(0)
    return out


def reference_normalised(x):
    x = np.asarray(x, dtype=np.float32)
    return x / np.linalg.norm(x, axis=1, keepdims=True)


def adversarial_rows(rng, n, d):
    """float32 rows [n][d] whose packed form exercises every term of the bound."""
    kind = rng.integers(0, 5, size=n)
    x = rng.standard_normal((n, d))
    mag = 10.0 ** rng.uniform(-7, 0, size=(n, d))                    # mixed magnitudes: many |u_i| < 2^-11 (lo subnormal), some < 2^-22
    x = np.where(kind[:, None] == 1, x * mag, x)
    x = np.where(kind[:, None] == 2, x * 1e30, x)                     # large norms (the squares overflow float32, not float64)
    dom = np.zeros((n, d))
    dom[np.arange(n), rng.integers(0, d, size=n)] = 1e4
    x = np.where(kind[:, None] == 3, x * 1e-3 + dom, x)               # one dominant element: the rest of the row is tiny relative to it
    x = np.where(kind[:, None] == 4, np.abs(x), x)                    # all positive: large cosines, distances near 0
    return x.astype(np.float32)
