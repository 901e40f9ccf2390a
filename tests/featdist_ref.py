"""TEST INFRASTRUCTURE: the float64 reference and error bound of the feature-distance kernel (csrc/b2t_tracker.cu, feat_dist_kernel;
C ABI b2t_feature_distance), StrongSORT's matching.embedding_distance(metric='euclidean').

The kernel sums ((double)a_k - (double)b_k)^2 over k in order, each operation rounded once (no FMA), then takes the square root.
With u = 2^-53 and gamma_k = k u / (1 - k u):
  * a float32 value is exact in float64; the difference d_k is rounded at most once: d_k (1 + e1), |e1| <= u;
  * the square is rounded once: d_k^2 (1 + e1)^2 (1 + e2);
  * D terms summed in order: each term picks up at most D - 1 further roundings, so the sum is S (1 + t), |t| <= gamma_{D+2};
  * sqrt(S (1 + t)) (1 + e3) = dist (1 + t') with |t'| <= (1 + gamma_{D+2})(1 + u) - 1 <= gamma_{D+3}  (sqrt(1 + t) lies between
    1 - |t| and 1 + |t| / 2).
So |kernel - dist| <= gamma_{D+3} * dist.  The reference ``exact`` evaluates the same difference form in extended precision
(np.longdouble, 64-bit significand); its own error, gamma'_{D+3} * dist with u' = 2^-64, is added to the bound."""
import numpy as np

U = 2.0 ** -53
U_REF = float(np.finfo(np.longdouble).eps) / 2


def gamma(k, u=U):
    return k * u / (1 - k * u)


def exact(a, b):
    """(n, m) extended-precision distances between the float32 rows of a (n, D) and b (m, D)."""
    a = np.asarray(a, np.float32).astype(np.longdouble)
    b = np.asarray(b, np.float32).astype(np.longdouble)
    out = np.zeros((a.shape[0], b.shape[0]), np.longdouble)
    for i in range(a.shape[0]):
        d = a[i][None, :] - b
        out[i] = np.sqrt((d * d).sum(axis=1))
    return out


def bound(ex, D):
    """The derived bound on |kernel - exact| (float64), plus the reference's own error."""
    ex = np.asarray(ex, np.float64)
    return (gamma(D + 3) + gamma(D + 3, U_REF)) * ex


def check(got, ex, D, what="feature distance"):
    got = np.asarray(got, np.float64)
    assert got.shape == ex.shape, "%s: shape %s != %s" % (what, got.shape, ex.shape)
    assert np.isfinite(got).all(), "%s: non-finite output" % what
    assert (got >= 0).all(), "%s: negative output" % what
    err = np.abs(got.astype(np.longdouble) - ex).astype(np.float64)
    b = bound(ex, D)
    bad = err > b
    assert not bad.any(), "%s: %d outputs beyond the bound, worst err/bound %.3g at %s" % (
        what, int(bad.sum()), float((err / np.maximum(b, 1e-300)).max()), np.argwhere(bad)[0])
    return float((err[b > 0] / b[b > 0]).max()) if (b > 0).any() else 0.0
