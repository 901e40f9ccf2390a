"""TEST INFRASTRUCTURE ONLY -- CPU restatement of the reference's ECC camera-motion estimator (``GMC(method='ecc')``).

Follows ``tracker/botsort.py:78-109`` (``GMC.applyEcc``) and the ``cv2.findTransformECC(template, image, H, MOTION_EUCLIDEAN,
(COUNT | EPS, 100, 1e-5), None, 1)`` call it makes, in NumPy, so that the CUDA kernels (csrc/b2t_ecc.cu) have something to be
compared with stage by stage.  The arithmetic of each OpenCV call was recovered by probing cv2 (4.13) with seeded inputs;
``tests/test_oracle_ecc.py`` re-checks every stage against the cv2 call and the whole estimate against the UNMODIFIED reference
class (tests/golden/ecc.npz).

Stage                          reference / cv2 call                            restatement      parity with cv2
gray                           cvtColor(BGR2GRAY), 15-bit luma                 prepare()        bit-exact
3 x 3 blur, sigma 1.5, uint8   GaussianBlur((3, 3), 1.5): fixed point, taps    prepare()        bit-exact
                               (79, 98, 79) / 256 per pass, rows then columns,
                               (v + 2^15) >> 16, BORDER_REFLECT_101
1/ds resize                    resize(INTER_LINEAR, 8-bit): 2 x 2 mean for an  prepare()        bit-exact
                               exact half, 11-bit taps otherwise
gradients                      filter2D([-0.5, 0, 0.5]) and its transpose,     gradients()      exact (halves of integers)
                               BORDER_REFLECT_101 (0 on the first / last column)
warp                           warpAffine(INTER_LINEAR | WARP_INVERSE_MAP),    warp_linear()    bit-exact (fp32 taps summed in
                               source coordinate in 1/32 px: AB_BITS 10,                        the order w00, w01, w10, w11)
                               round-half-even of M * x * 1024, + 16, >> 5
mask                           warpAffine(ones, INTER_NEAREST), + 512, >> 10   warp_nearest()   bit-exact
ECC step                       meanStdDev, dot products, 3 x 3 inverse,        ecc()            fp64 sums over the fp32 pixels
                               lambda, delta p, map update                                      (OpenCV sums fp32 products in
                                                                                                SIMD blocks): H to ~1e-7

Quirks of the reference that are reproduced (DESIGN.md, q17):
  * the template is the sequence's FIRST frame and is never replaced: every later frame is aligned to frame 1;
  * the warp is in down-scaled pixels (unlike the ORB path, the translation is not multiplied back by ``downscale``);
  * outside the warped mask the zero-mean image keeps its raw warped values (``subtract(..., mask)`` leaves them), so the image
    projection and the Hessian include border pixels whose bilinear taps reach into the image while the nearest one does not;
  * OpenCV 4.13 tests lambda_d <= 0 before it tests rho for NaN: a flat frame (rho = 0 / 0, lambda_d = 0) fails with "The algorithm
    stopped before its convergence", not with "NaN encountered" (measured: tests/golden/ecc.npz case 3);
  * on an exception (lambda_d <= 0, NaN rho) the returned H is the map after the last completed update (findTransformECC updates
    the caller's float32 array in place).
"""
import numpy as np

FIRST_FRAME, CONVERGED, ITER_CAP, FAILED_NAN, FAILED_LAMBDA = 1, 2, 4, 8, 16    # include/b200track.h B2T_ECC_*
BLUR3 = np.array([79, 98, 79], np.int64)            # GaussianBlur((3, 3), 1.5) on uint8: taps in 1/256


def gray(frame_bgr):
    f = frame_bgr.astype(np.int64)
    return ((f[..., 0] * 3735 + f[..., 1] * 19235 + f[..., 2] * 9798 + (1 << 14)) >> 15).astype(np.uint8)


def blur3(g):
    """cv2.GaussianBlur(g, (3, 3), 1.5) for uint8 g: separable fixed point, rows then columns, BORDER_REFLECT_101."""
    h, w = g.shape
    p = np.pad(g.astype(np.int64), 1, mode="reflect")
    r = sum(BLUR3[j] * p[:, j:j + w] for j in range(3))
    v = sum(BLUR3[i] * r[i:i + h] for i in range(3))
    return ((v + (1 << 15)) >> 16).astype(np.uint8)


def prepare(frame_bgr, downscale=2):
    """GMC.applyEcc's preparation (botsort.py:81-90): gray; for downscale > 1 the 3 x 3 blur and cv2.resize to (w // ds, h // ds)."""
    g = gray(frame_bgr)
    if downscale <= 1:
        return g
    b = blur3(g)
    h, w = b.shape
    if downscale == 2 and h % 2 == 0 and w % 2 == 0:
        a = b.astype(np.int32)
        return ((a[0::2, 0::2] + a[0::2, 1::2] + a[1::2, 0::2] + a[1::2, 1::2] + 2) >> 2).astype(np.uint8)
    from oracle import preprocess as P
    return P.resize_linear_u8(b[..., None], (w // downscale, h // downscale))[..., 0]


def gradients(img):
    """filter2D with (-0.5, 0, 0.5) along x and along y, BORDER_REFLECT_101 (the reflected neighbour cancels: 0 on the edges)."""
    a = img.astype(np.float32)
    gx = np.zeros_like(a); gy = np.zeros_like(a)
    gx[:, 1:-1] = np.float32(0.5) * (a[:, 2:] - a[:, :-2])
    gy[1:-1, :] = np.float32(0.5) * (a[2:, :] - a[:-2, :])
    return gx, gy


def _coords(M, h, w, nearest):
    """warpAffine's fixed-point source coordinates for the destination grid (WARP_INVERSE_MAP: M maps destination to source)."""
    M = np.asarray(M, np.float32).astype(np.float64)
    ys, xs = np.mgrid[0:h, 0:w]
    ad = np.rint(M[0, 0] * xs * 1024).astype(np.int64)
    bd = np.rint(M[1, 0] * xs * 1024).astype(np.int64)
    rd = 512 if nearest else 16
    X0 = np.rint((M[0, 1] * ys + M[0, 2]) * 1024).astype(np.int64) + rd
    Y0 = np.rint((M[1, 1] * ys + M[1, 2]) * 1024).astype(np.int64) + rd
    sh = 10 if nearest else 5
    return (X0 + ad) >> sh, (Y0 + bd) >> sh


def warp_linear(src, M):
    """cv2.warpAffine(src float32, M, src size, INTER_LINEAR | WARP_INVERSE_MAP), border 0."""
    h, w = src.shape
    X, Y = _coords(M, h, w, False)
    sx, sy = X >> 5, Y >> 5
    fx = (X & 31).astype(np.float32) / np.float32(32)
    fy = (Y & 31).astype(np.float32) / np.float32(32)
    pad = np.zeros((h + 2, w + 2), np.float32)
    pad[1:-1, 1:-1] = src

    def at(yy, xx):
        ok = (yy >= -1) & (yy <= h) & (xx >= -1) & (xx <= w)
        return np.where(ok, pad[np.clip(yy + 1, 0, h + 1), np.clip(xx + 1, 0, w + 1)], np.float32(0))
    one = np.float32(1)
    return (at(sy, sx) * ((one - fy) * (one - fx)) + at(sy, sx + 1) * ((one - fy) * fx)
            + at(sy + 1, sx) * (fy * (one - fx)) + at(sy + 1, sx + 1) * (fy * fx)).astype(np.float32)


def warp_nearest_mask(h, w, M):
    """cv2.warpAffine(ones uint8, M, (w, h), INTER_NEAREST | WARP_INVERSE_MAP), border 0: 1 where the source pixel exists."""
    X, Y = _coords(M, h, w, True)
    return ((X >= 0) & (X < w) & (Y >= 0) & (Y < h)).astype(np.uint8)


def _f32(v):
    return np.float64(np.float32(v))


def inv3_f32(Hf):
    """Mat::inv() of a float32 3 x 3 (closed form in double from the float entries, rounded to float32)."""
    m = Hf.astype(np.float64)
    d = (m[0, 0] * (m[1, 1] * m[2, 2] - m[1, 2] * m[2, 1]) - m[0, 1] * (m[1, 0] * m[2, 2] - m[1, 2] * m[2, 0])
         + m[0, 2] * (m[1, 0] * m[2, 1] - m[1, 1] * m[2, 0]))
    if d == 0:
        return np.zeros((3, 3), np.float64)
    d = 1.0 / d
    t = np.array([[m[1, 1] * m[2, 2] - m[1, 2] * m[2, 1], m[0, 2] * m[2, 1] - m[0, 1] * m[2, 2], m[0, 1] * m[1, 2] - m[0, 2] * m[1, 1]],
                  [m[1, 2] * m[2, 0] - m[1, 0] * m[2, 2], m[0, 0] * m[2, 2] - m[0, 2] * m[2, 0], m[0, 2] * m[1, 0] - m[0, 0] * m[1, 2]],
                  [m[1, 0] * m[2, 1] - m[1, 1] * m[2, 0], m[0, 1] * m[2, 0] - m[0, 0] * m[2, 1], m[0, 0] * m[1, 1] - m[0, 1] * m[1, 0]]]) * d
    return t.astype(np.float32).astype(np.float64)


def sums(tmpl, img, gx, gy, M):
    """The 21 sums one iteration needs, in fp64 over fp32 pixel values (the kernel accumulates the same ones):
    n, S_I, S_II, S_T, S_TT, S_TI over the mask; S_JI (3) over all pixels; S_J, S_JT (3 each) over the mask; S_JJ (6, all pixels)."""
    h, w = tmpl.shape
    I = warp_linear(img.astype(np.float32), M)
    GX, GY = warp_linear(gx, M), warp_linear(gy, M)
    m = warp_nearest_mask(h, w, M).astype(bool)
    T = tmpl.astype(np.float32)
    c, s = np.float32(M[0][0]), np.float32(M[1][0])
    ys, xs = np.mgrid[0:h, 0:w].astype(np.float32)
    hatX = -(xs * s) - (ys * c)
    hatY = (xs * c) - (ys * s)
    J = [GX * hatX + GY * hatY, GX, GY]
    J = [j.astype(np.float64) for j in J]
    I64, T64 = I.astype(np.float64), T.astype(np.float64)
    out = dict(n=float(m.sum()), SI=I64[m].sum(), SII=(I64 * I64)[m].sum(), ST=T64[m].sum(), STT=(T64 * T64)[m].sum(),
               STI=(T64 * I64)[m].sum(),
               SJI=np.array([(j * I64).sum() for j in J]), SJ=np.array([j[m].sum() for j in J]),
               SJT=np.array([(j * T64)[m].sum() for j in J]),
               SJJ=np.array([[(J[a] * J[b]).sum() for b in range(3)] for a in range(3)]))
    return out


def step(sm, M):
    """One findTransformECC iteration from the sums.  Returns (new map float32 (2, 3), rho, flag): flag 0, FAILED_LAMBDA or FAILED_NAN
    (the map is then the input map)."""
    n = sm["n"]
    im, tm = sm["SI"] / n, sm["ST"] / n
    istd = np.sqrt(max(sm["SII"] / n - im * im, 0.0))
    tstd = np.sqrt(max(sm["STT"] / n - tm * tm, 0.0))
    imf, tmf = _f32(im), _f32(tm)
    tnorm, inorm = np.sqrt(n * tstd * tstd), np.sqrt(n * istd * istd)
    Hf = np.vectorize(_f32)(sm["SJJ"])
    Hi = inv3_f32(Hf)
    corr = sm["STI"] - imf * sm["ST"] - tmf * sm["SI"] + n * tmf * imf
    with np.errstate(divide="ignore", invalid="ignore"):
        rho = corr / (inorm * tnorm)
    iproj = sm["SJI"] - imf * sm["SJ"]
    tproj = sm["SJT"] - tmf * sm["SJ"]
    ipf, tpf = np.vectorize(_f32)(iproj), np.vectorize(_f32)(tproj)
    iph = np.vectorize(_f32)(Hi @ ipf)
    lam_n = inorm * inorm - float(ipf @ iph)
    lam_d = corr - float(tpf @ iph)
    if lam_d <= 0.0:
        return M, rho, FAILED_LAMBDA
    if np.isnan(rho):                                   # after the lambda test: see the module docstring
        return M, rho, FAILED_NAN
    lam = lam_n / lam_d
    ep = np.vectorize(_f32)(lam * tproj - iproj)
    dp = np.vectorize(_f32)(Hi @ ep)
    M = np.array(M, np.float32)
    theta = dp[0] + np.arcsin(np.float64(M[1, 0]))
    M[0, 2] = np.float32(M[0, 2] + np.float32(dp[1]))
    M[1, 2] = np.float32(M[1, 2] + np.float32(dp[2]))
    M[0, 0] = M[1, 1] = np.float32(np.cos(theta))
    M[1, 0] = np.float32(np.sin(theta))
    M[0, 1] = -M[1, 0]
    return M, rho, 0


def ecc(tmpl, img, max_iter=100, eps=1e-5, trace=None):
    """findTransformECC(tmpl, img, eye(2, 3, float32), MOTION_EUCLIDEAN, (COUNT | EPS, max_iter, eps), None, 1).
    Returns (H float32 (2, 3), iterations run, flags, final rho).  ``trace`` (a list) receives (rho, map) per iteration."""
    M = np.eye(2, 3, dtype=np.float32)
    gx, gy = gradients(img)
    rho, last = -1.0, -eps
    it = 0
    while it < max_iter and abs(rho - last) >= eps:
        it += 1
        sm = sums(tmpl, img, gx, gy, M)
        M2, r, fl = step(sm, M)
        last, rho = rho, r
        if fl:
            return M, it, fl, rho
        M = M2
        if trace is not None:
            trace.append((rho, M.copy()))
    return M, it, (CONVERGED if abs(rho - last) < eps else ITER_CAP), rho


class EccOracle:
    """GMC(method='ecc', downscale).apply restated: the first frame becomes the template (never replaced, q17)."""

    def __init__(self, downscale=2, max_iter=100, eps=1e-5):
        self.downscale, self.max_iter, self.eps = max(1, int(downscale)), max_iter, eps
        self.template = None

    def apply(self, frame_bgr):
        """-> (H float32 (2, 3), iterations, flags, rho)"""
        p = prepare(frame_bgr, self.downscale)
        if self.template is None:
            self.template = p
            return np.eye(2, 3, dtype=np.float32), 0, FIRST_FRAME, 0.0
        return ecc(self.template, p, self.max_iter, self.eps)
