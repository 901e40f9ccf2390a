"""TEST INFRASTRUCTURE: the ORB camera-motion stage checks (csrc/b2t_gmc.cu) shared by the GPU tier (tests/test_gpu_gmc_stages.py)
and the simulator tier (tests/test_hostsim_gmc_stages.py).  ``Checker.frame`` checks one estimate call of every sequence from the
workspace the kernels left, against oracle/gmc.py, and returns the failed stages by name instead of asserting (so that an
injected bug can be shown to fail at its stage):

  keypoints   FAST + mask + ORB border, first max_kp in row-major order, and the descriptors: bit for bit
  flags       FIRST_FRAME, TRUNCATED (iff the oracle found more than max_kp corners)
  ratio       the count after the ratio and spatial tests (stat 2): exact (integer distances and coordinates)
  sigma       the estimator's point set after the one-sided 2.5 sigma test, in order, against ``filter_matches``: only points
              within the sigma test's rounding band (derived from block_sum's depth) may differ
  ransac      best hypothesis (stat 6) and its inlier count (stat 4) on the device's own point set: exact
  fit         the warp against the least-squares similarity on those inliers, within a derived bound"""
import math

import numpy as np

from b200track import _lib as L
from b200track import gmc as G
from oracle import gmc as OG

U = 2.0 ** -53
EST_THREADS = 1024


def gamma(n):
    return n * U / (1 - n * U)


def block_depth(n):
    """block_sum's depth over n terms: ceil(n / 1024) sequential adds per thread, 5 butterfly levels, 32 warps in order."""
    return -(-max(n, 1) // EST_THREADS) + 5 + EST_THREADS // 32


def ransac_best(pts):
    """(inlier count, hypothesis) of ransac_kernel: most inliers, ties to the lowest hypothesis; (0, -1) for n <= 4."""
    n = len(pts)
    if n <= 4:
        return 0, -1
    src, dst = pts[:, :2].astype(np.float64), pts[:, 2:].astype(np.float64)
    best, bt = -1, -1
    for t in range(OG.RANSAC_HYPOTHESES):
        i, j = OG.lcg_pair(t, n)
        m = OG.similarity_from_pair(src[i], src[j], dst[i], dst[j])
        if m is None:
            continue
        a, b, tx, ty = m
        ex = a * src[:, 0] - b * src[:, 1] + tx - dst[:, 0]
        ey = b * src[:, 0] + a * src[:, 1] + ty - dst[:, 1]
        c = int((ex * ex + ey * ey < 9.0).sum())
        if c > best:
            best, bt = c, t
    return max(best, 0), bt


def fit_with_bound(src, dst, ds):
    """The least-squares similarity on (src, dst) as fit_kernel computes it, and a bound on |kernel - this| per warp entry.  The
    coordinate sums are sums of integers (exact), so the means are the same correctly rounded quotients; the centred terms are the
    same roundings; only the sums of the centred products differ, by at most gamma_D + gamma_P of their absolute sums (D: block_sum's
    depth, P: NumPy's pairwise depth)."""
    n = len(src)
    ms, md = src.mean(0), dst.mean(0)
    x, y, u, v = src[:, 0] - ms[0], src[:, 1] - ms[1], dst[:, 0] - md[0], dst[:, 1] - md[1]
    ta, tb, td = x * u + y * v, x * v - y * u, x * x + y * y
    g = gamma(block_depth(n)) + gamma(int(math.ceil(math.log2(max(n, 2)))) + 8)
    na, nb, den = ta.sum(), tb.sum(), td.sum()
    ea, eb, ed = (g * np.abs(t).sum() for t in (ta, tb, td))
    a, b = na / den, nb / den
    da = ((ea + abs(a) * ed) / (den - ed) + 2 * U * abs(a)) * 1.01
    db = ((eb + abs(b) * ed) / (den - ed) + 2 * U * abs(b)) * 1.01
    tx = (md[0] - (a * ms[0] - b * ms[1])) * ds
    ty = (md[1] - (b * ms[0] + a * ms[1])) * ds
    etx = ((abs(ms[0]) * da + abs(ms[1]) * db) * 1.01 + 8 * U * (abs(md[0]) + abs(a * ms[0]) + abs(b * ms[1]))) * ds
    ety = ((abs(ms[0]) * db + abs(ms[1]) * da) * 1.01 + 8 * U * (abs(md[1]) + abs(b * ms[0]) + abs(a * ms[1]))) * ds
    H = np.array([[a, -b, tx], [b, a, ty]])
    E = np.array([[da, db, etx], [db, da, ety]])
    return H, E


def sigma_test(prev_xy, cur_xy, i1, d1, d2, width, height):
    """filter_matches with its intermediate results: (q after the ratio + spatial tests, keep mask of the sigma test, band mask:
    points whose sigma-test margin is within the kernel's rounding of the mean and std)."""
    ok = d1.astype(np.float64) < 0.9 * d2.astype(np.float64)
    dist = prev_xy.astype(np.float64) - cur_xy[i1].astype(np.float64)
    ok &= (np.abs(dist[:, 0]) < 0.25 * width) & (np.abs(dist[:, 1]) < 0.25 * height)
    q = np.nonzero(ok)[0]
    if len(q) == 0:
        return q, np.zeros(0, bool), np.zeros(0, bool)
    sd = dist[q]
    n = len(q)
    mean, std = sd.mean(0), sd.std(0)
    g = gamma(block_depth(n)) + gamma(int(math.ceil(math.log2(max(n, 2)))) + 8)
    e_mean = g * np.abs(sd).sum(0) / n + 4 * U * np.abs(mean)
    e2 = ((sd - mean) ** 2).sum(0)
    e_var = (g * e2 + 2 * np.abs(sd - mean).sum(0) * e_mean) / n + 4 * U * e2 / n
    e_std = np.where(std > 0, e_var / np.maximum(std, 1e-300) / 2, np.sqrt(e_var)) + 4 * U * std
    band_w = 2 * (e_mean + 2.5 * e_std) + 8 * U * (np.abs(sd) + np.abs(mean) + 2.5 * std)
    margin = np.abs((sd - mean) - 2.5 * std)
    keep = np.all((sd - mean) < 2.5 * std, axis=1)
    band = np.any(margin <= band_w, axis=1)
    return q, keep, band


class Checker:
    """Per-sequence oracle state across the frames of one run: the previous (truncated) key points and descriptors."""

    def __init__(self, n_seq, ds, max_kp):
        self.S, self.ds, self.max_kp = n_seq, ds, max_kp
        self.prev = [None] * n_seq
        self.report = dict(sigma_band=0, points=0, worst_fit=0.0)

    def reset(self):
        self.prev = [None] * self.S

    def frame(self, frames, dets, warps, stat, ws, layout):
        """dets[s]: the detections the mask uses (already thresholded) or None.  Returns [(seq, stage, detail)]."""
        bad = []
        for s in range(self.S):
            g, xs, ys, desc = OG.GMCOracle(self.ds).stages(frames[s], dets[s])
            trunc = len(xs) > self.max_kp
            xs, ys, desc = xs[:self.max_kp], ys[:self.max_kp], desc[:self.max_kp]
            state = np.frombuffer(ws, np.int32, 16, s * layout["stride"] + layout["state"])
            buf = (int(state[0]) - 1) & 1
            kx, ky, kd = G.unpack_keypoints(ws, layout, s, buf, int(state[1 + buf]), self.max_kp)
            if not (np.array_equal(kx, xs) and np.array_equal(ky, ys) and np.array_equal(kd, desc)) or stat[s, 0] != len(xs):
                bad.append((s, "keypoints", (len(kx), len(xs))))
            first = self.prev[s] is None
            want = (L.GMC_FIRST_FRAME if first else 0) | (L.GMC_TRUNCATED if trunc else 0)
            if stat[s, 5] & (L.GMC_FIRST_FRAME | L.GMC_TRUNCATED) != want:
                bad.append((s, "flags", (int(stat[s, 5]), want)))
            prev, self.prev[s] = self.prev[s], (xs, ys, desc)
            if first:
                if not np.array_equal(warps[s], np.eye(2, 3)):
                    bad.append((s, "fit", "first frame is not the identity"))
                continue
            pxy = np.stack([prev[0], prev[1]], 1)
            cxy = np.stack([xs, ys], 1)
            if len(prev[0]) == 0 or len(xs) < 2:
                q, keep, band = np.zeros(0, int), np.zeros(0, bool), np.zeros(0, bool)
            else:
                i1, d1, _, d2 = OG.knn2(prev[2], desc)
                q, keep, band = sigma_test(pxy, cxy, i1, d1, d2, g.shape[1], g.shape[0])
            if stat[s, 2] != len(q):
                bad.append((s, "ratio", (int(stat[s, 2]), len(q))))
                continue
            n_sigma = int(stat[s, 3])
            pts = np.frombuffer(ws, np.float32, 4 * n_sigma, s * layout["stride"] + layout["pts"] + self.max_kp * 16).reshape(n_sigma, 4)
            exp = np.concatenate([pxy[q], cxy[i1[q]]], 1).astype(np.float32) if len(q) else np.zeros((0, 4), np.float32)
            self.report["sigma_band"] += int(band.sum())
            self.report["points"] += len(q)
            if not band.any():
                if not np.array_equal(pts, exp[keep]):
                    bad.append((s, "sigma", (n_sigma, int(keep.sum()))))
                    continue
            else:                                          # points in the band may go either way; all others must agree
                got = {tuple(p) for p in pts.tolist()}
                if any((tuple(p) in got) != k for p, k, b in zip(exp.tolist(), keep, band) if not b):
                    bad.append((s, "sigma", "outside the band"))
                    continue
            cnt, t = ransac_best(pts)
            if (int(stat[s, 4]), int(stat[s, 6])) != (cnt, t):
                bad.append((s, "ransac", ((int(stat[s, 4]), int(stat[s, 6])), (cnt, t))))
                continue
            if cnt >= 2:
                src, dst = pts[:, :2].astype(np.float64), pts[:, 2:].astype(np.float64)
                a, b, tx, ty = OG.similarity_from_pair(src[OG.lcg_pair(t, len(pts))[0]], src[OG.lcg_pair(t, len(pts))[1]],
                                                       dst[OG.lcg_pair(t, len(pts))[0]], dst[OG.lcg_pair(t, len(pts))[1]])
                ex = a * src[:, 0] - b * src[:, 1] + tx - dst[:, 0]
                ey = b * src[:, 0] + a * src[:, 1] + ty - dst[:, 1]
                inl = ex * ex + ey * ey < 9.0
                H, E = fit_with_bound(src[inl], dst[inl], self.ds)
                err = np.abs(warps[s] - H)
                self.report["worst_fit"] = max(self.report["worst_fit"], float((err / E).max()))
                if not (err <= E).all():
                    bad.append((s, "fit", float((err / E).max())))
            elif not np.array_equal(warps[s], np.eye(2, 3)):
                bad.append((s, "fit", "too few points but not the identity"))
        return bad


def thresholded(dets, counts, thresh):
    """Per sequence: the detections the mask uses (score >= thresh) or None."""
    if dets is None:
        return [None] * 1
    return [d[:c][d[:c, 4] >= np.float32(thresh)] for d, c in zip(dets, counts)]


def many_boxes(h, w, n=400, seed=0):
    """n tall boxes over every row of an (h, w) frame -- more than the 256 a row caches -- plus boxes with negative and out-of-frame
    corners, and some below the threshold 0.2."""
    rng = np.random.default_rng(seed)
    x0 = rng.uniform(-20, w, n)
    box = np.stack([x0, rng.uniform(-40, 0.3 * h, n), x0 + rng.uniform(0.5, 3, n), rng.uniform(0.7 * h, h + 40, n)], 1)
    extra = np.array([[-30, -30, 0.1 * w, 0.1 * h], [0.9 * w, 0.9 * h, w + 50, h + 50], [-5.5, 0.4 * h, 0.3 * w, 0.5 * h]])
    box = np.concatenate([box, extra])
    score = np.where(np.arange(len(box)) % 7 == 3, 0.1, 0.9)
    return np.concatenate([box, score[:, None], np.zeros((len(box), 1))], 1).astype(np.float32)
