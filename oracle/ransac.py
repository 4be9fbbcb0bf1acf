"""TEST INFRASTRUCTURE ONLY.  Pure-NumPy restatement of OpenCV's RANSACPointSetRegistrator (calib3d ptsetreg.cpp)
for cv2.findHomography / cv2.estimateAffinePartial2D as the reference calls them (fastmot/flow.py:215-279), and of the
serial per-track loop around them.  It documents what csrc/klt_ransac.cu computes and is itself pinned against cv2
in tests/test_oracle_ransac.py:

- the RNG (64-bit multiply-with-carry seeded with (uint64)-1), getSubset's redraw rule and its 10000 attempts,
  checkSubset, "first strictly better wins" and RANSACUpdateNumIters, statement by statement;
- the error of a point is OpenCV's computeError in float32 (model rounded to float, float arithmetic, no FMA);
- 4-point homography hypotheses use the kernel's normalised exact 8x8 solve (OpenCV takes the smallest eigenvector
  of the 9x9 normal matrix: the two differ at rounding level only);
- the final DLT and the Levenberg-Marquardt refinement (levmarq.cpp: lambda schedule 0.25 / 0.75, at most 10
  iterations) run in float64;
- findHomography's mask is recomputed under the refined model over every point; estimateAffinePartial2D's mask is
  the best hypothesis's.
"""
import math
from dataclasses import dataclass, field

import numpy as np

f32 = np.float32
DBL_MIN = np.finfo(np.float64).tiny
DBL_EPSILON = np.finfo(np.float64).eps
FLT_EPSILON = float(np.finfo(np.float32).eps)
U64 = (1 << 64) - 1


class CvRng:
    """cv::RNG: state = (uint32)state * 4164903690 + (state >> 32)."""

    def __init__(self, state=U64):
        self.state = state
        self.draws = 0

    def next(self):
        self.state = ((self.state & 0xffffffff) * 4164903690 + (self.state >> 32)) & U64
        self.draws += 1
        return self.state & 0xffffffff

    def uniform(self, a, b):
        return a if a == b else self.next() % (b - a) + a


def get_subset(m, k, rng, check=None, max_attempts=10000):
    """Indices of k distinct points (a repeated index is redrawn at once); when the whole subset fails `check` every
    index is drawn again, at most max_attempts times.  None when no subset passed."""
    for _ in range(max_attempts):
        idx = []
        for _ in range(k):
            v = rng.uniform(0, m)
            while v in idx:
                v = rng.uniform(0, m)
            idx.append(v)
        if check is None or check(idx):
            return idx
    return None


def update_num_iters(p, ep, k, niters):
    """RANSACUpdateNumIters."""
    p = min(max(p, 0.), 1.)
    ep = min(max(ep, 0.), 1.)
    num = max(1. - p, DBL_MIN)
    denom = 1. - (1. - ep) ** k
    if denom < DBL_MIN:
        return 0
    num, denom = math.log(num), math.log(denom)
    return niters if denom >= 0 or -num >= niters * (-denom) else int(np.rint(num / denom))


# ------------------------------------------------------------------------------------------------ homography
def _have_collinear(pts):
    """haveCollinearPoints(count=4): is the last point on a line through two earlier ones?  Differences in float."""
    i = len(pts) - 1
    for j in range(i):
        dx1, dy1 = float(pts[j, 0] - pts[i, 0]), float(pts[j, 1] - pts[i, 1])
        for k in range(j):
            dx2, dy2 = float(pts[k, 0] - pts[i, 0]), float(pts[k, 1] - pts[i, 1])
            if abs(dx2 * dy1 - dy2 * dx1) <= FLT_EPSILON * (abs(dx1) + abs(dy1) + abs(dx2) + abs(dy2)):
                return True
    return False


def _det3(a, b, c):
    a, b, c = a.astype(np.float64), b.astype(np.float64), c.astype(np.float64)
    return a[0] * (b[1] - c[1]) - a[1] * (b[0] - c[0]) + (b[0] * c[1] - b[1] * c[0])


def homography_check_subset(s, d):
    """HomographyEstimatorCallback::checkSubset: no collinear triple (last point) in either set, and the four
    triangles keep (or all flip) their orientation."""
    if _have_collinear(s) or _have_collinear(d):
        return False
    neg = 0
    for t in ((0, 1, 2), (1, 2, 3), (0, 2, 3), (0, 1, 3)):
        neg += _det3(s[t[0]], s[t[1]], s[t[2]]) * _det3(d[t[0]], d[t[1]], d[t[2]]) < 0
    return neg == 0 or neg == 4


def solve_dense(A, b):
    """Gaussian elimination with partial pivoting (the kernel's solve_dense); None when singular."""
    A, b = A.astype(np.float64).copy(), b.astype(np.float64).copy()
    n = len(b)
    for c in range(n):
        piv = c + int(np.argmax(np.abs(A[c:, c])))
        if not abs(A[piv, c]) > 0.0:
            return None
        if piv != c:
            A[[c, piv]] = A[[piv, c]]
            b[[c, piv]] = b[[piv, c]]
        f = A[c + 1:, c] / A[c, c]
        A[c + 1:, c:] -= f[:, None] * A[c, c:]
        b[c + 1:] -= f * b[c]
    x = np.zeros(n)
    for r in range(n - 1, -1, -1):
        x[r] = (b[r] - A[r, r + 1:] @ x[r + 1:]) / A[r, r]
    return x


def _normalisation(M, m):
    M, m = M.astype(np.float64), m.astype(np.float64)
    cM, cm = M.mean(0), m.mean(0)
    sM, sm = np.abs(M - cM).sum(0), np.abs(m - cm).sum(0)
    if (np.abs(np.concatenate([sM, sm])) < DBL_EPSILON).any():
        return None
    return cM, len(M) / sM, cm, len(m) / sm


def _denormalise(H0, cM, sM, cm, sm):
    inv_hnorm = np.array([[1 / sm[0], 0, cm[0]], [0, 1 / sm[1], cm[1]], [0, 0, 1.]])
    hnorm2 = np.array([[sM[0], 0, -cM[0] * sM[0]], [0, sM[1], -cM[1] * sM[1]], [0, 0, 1.]])
    H = inv_hnorm @ H0 @ hnorm2
    return H / H[2, 2]


def homography_from4(M, m):
    """4-point hypothesis: OpenCV's normalisation, then the exact 8x8 solve of the normalised DLT (h33 = 1)."""
    nrm = _normalisation(M, m)
    if nrm is None:
        return None
    cM, sM, cm, sm = nrm
    X, Y = ((M - cM) * sM).T
    x, y = ((m - cm) * sm).T
    A = np.zeros((8, 8))
    A[0::2, 0], A[0::2, 1], A[0::2, 2], A[0::2, 6], A[0::2, 7] = X, Y, 1, -x * X, -x * Y
    A[1::2, 3], A[1::2, 4], A[1::2, 5], A[1::2, 6], A[1::2, 7] = X, Y, 1, -y * X, -y * Y
    b = np.empty(8)
    b[0::2], b[1::2] = x, y
    h = solve_dense(A, b)
    if h is None:
        return None
    return _denormalise(np.append(h, 1.).reshape(3, 3), cM, sM, cm, sm)


def homography_dlt(M, m):
    """HomographyEstimatorCallback::runKernel on n >= 4 points: smallest eigenvector of the normalised 9x9 LtL."""
    nrm = _normalisation(M, m)
    if nrm is None:
        return None
    cM, sM, cm, sm = nrm
    X, Y = ((M - cM) * sM).T
    x, y = ((m - cm) * sm).T
    o, z = np.ones_like(X), np.zeros_like(X)
    Lx = np.stack([X, Y, o, z, z, z, -x * X, -x * Y, -x], 1)
    Ly = np.stack([z, z, z, X, Y, o, -y * X, -y * Y, -y], 1)
    w, V = np.linalg.eigh(Lx.T @ Lx + Ly.T @ Ly)
    return _denormalise(V[:, 0].reshape(3, 3), cM, sM, cm, sm)


def homography_error(H, M, m):
    """HomographyEstimatorCallback::computeError: float model (H[0..7]), float arithmetic."""
    Hf = np.asarray(H, np.float64).ravel()[:8].astype(f32)
    X, Y = M[:, 0].astype(f32), M[:, 1].astype(f32)
    ww = f32(1) / (Hf[6] * X + Hf[7] * Y + f32(1))
    dx = (Hf[0] * X + Hf[1] * Y + Hf[2]) * ww - m[:, 0].astype(f32)
    dy = (Hf[3] * X + Hf[4] * Y + Hf[5]) * ww - m[:, 1].astype(f32)
    return dx * dx + dy * dy


# ------------------------------------------------------------------------------------------------ affine partial
def affine_partial_from2(M, m):
    """AffinePartial2DEstimatorCallback::runKernel: the closed-form similarity through two matches (2x3, float64)."""
    x1, y1, x2, y2 = (float(v) for v in (M[0, 0], M[0, 1], M[1, 0], M[1, 1]))
    X1, Y1, X2, Y2 = (float(v) for v in (m[0, 0], m[0, 1], m[1, 0], m[1, 1]))
    with np.errstate(divide="ignore", invalid="ignore"):
        d = np.float64(1.) / np.float64((x1 - x2) * (x1 - x2) + (y1 - y2) * (y1 - y2))
        S0 = d * ((X1 - X2) * (x1 - x2) + (Y1 - Y2) * (y1 - y2))
        S1 = d * ((Y1 - Y2) * (x1 - x2) - (X1 - X2) * (y1 - y2))
        S2 = d * ((Y1 - Y2) * (x1 * y2 - x2 * y1) - (X1 * y2 - X2 * y1) * (y1 - y2) - (X1 * x2 - X2 * x1) * (x1 - x2))
        S3 = d * (-(X1 - X2) * (x1 * y2 - x2 * y1) - (Y1 * x2 - Y2 * x1) * (x1 - x2) - (Y1 * y2 - Y2 * y1) * (y1 - y2))
    return np.array([[S0, -S1, S2], [S1, S0, S3]])


def affine_error(F, M, m, precision="float"):
    """Affine2DEstimatorCallback::computeError.  "float" (what OpenCV does, pinned in tests/test_oracle_ransac.py):
    model rounded to float, residual in float.  "double": residual in double, only the squared error rounded."""
    F = np.asarray(F, np.float64).ravel()
    with np.errstate(invalid="ignore", over="ignore"):
        if precision == "float":
            Ff = F.astype(f32)
            X, Y = M[:, 0].astype(f32), M[:, 1].astype(f32)
            a = Ff[0] * X + Ff[1] * Y + Ff[2] - m[:, 0].astype(f32)
            b = Ff[3] * X + Ff[4] * Y + Ff[5] - m[:, 1].astype(f32)
            return a * a + b * b
        X, Y = M[:, 0].astype(np.float64), M[:, 1].astype(np.float64)
        a = F[0] * X + F[1] * Y + F[2] - m[:, 0]
        b = F[3] * X + F[4] * Y + F[5] - m[:, 1]
        return (a * a + b * b).astype(f32)


# ------------------------------------------------------------------------------------------------ LM (levmarq.cpp)
def lm_refine(compute, x, max_iters=10):
    """LMSolverImpl::run: compute(x) -> (residuals, Jacobian).  Float64; stops on maxIters, |d|_inf < FLT_EPSILON or
    |r|_inf < FLT_EPSILON like OpenCV."""
    x = np.asarray(x, np.float64).copy()
    r, J = compute(x)
    S = float(r @ r)
    A, v = J.T @ J, J.T @ r
    D = np.diag(A).copy()
    lam, lc, it = 1., 0.75, 0
    while True:
        Ap = A + np.diag(lam * D)
        try:
            d = np.linalg.solve(Ap, v)
        except np.linalg.LinAlgError:
            d = np.linalg.pinv(Ap) @ v
        xd = x - d
        rd, _ = compute(xd)
        Sd = float(rd @ rd)
        dS = float(d @ (2 * v - A @ d))
        R = (S - Sd) / (dS if abs(dS) > DBL_EPSILON else 1.)
        if R > 0.75:
            lam *= 0.5
            if lam < lc:
                lam = 0.
        elif R < 0.25:
            t = float(d @ v)
            nu = min(max((Sd - S) / (t if abs(t) > DBL_EPSILON else 1.) + 2, 2.), 10.)
            if lam == 0:
                maxval = max(DBL_EPSILON, float(np.abs(np.diag(np.linalg.pinv(A))).max()))
                lam = lc = 1. / maxval
                nu *= 0.5
            lam *= nu
        if Sd < S:
            S, x = Sd, xd
            r, J = compute(x)
            A, v = J.T @ J, J.T @ r
        it += 1
        if not (it < max_iters and np.abs(d).max() >= FLT_EPSILON and np.abs(r).max() >= FLT_EPSILON):
            return x


def _affine_cb(M, m):
    M, m = M.astype(np.float64), m.astype(np.float64)

    def compute(h):
        ex = h[0] * M[:, 0] - h[1] * M[:, 1] + h[2] - m[:, 0]
        ey = h[1] * M[:, 0] + h[0] * M[:, 1] + h[3] - m[:, 1]
        o, z = np.ones(len(M)), np.zeros(len(M))
        J = np.concatenate([np.stack([M[:, 0], -M[:, 1], o, z], 1), np.stack([M[:, 1], M[:, 0], z, o], 1)])
        return np.concatenate([ex, ey]), J
    return compute


def _homography_cb(M, m):
    M, m = M.astype(np.float64), m.astype(np.float64)

    def compute(h):
        ww = h[6] * M[:, 0] + h[7] * M[:, 1] + 1.
        ww = np.where(np.abs(ww) > DBL_EPSILON, 1. / np.where(ww == 0, 1., ww), 0.)
        xi = (h[0] * M[:, 0] + h[1] * M[:, 1] + h[2]) * ww
        yi = (h[3] * M[:, 0] + h[4] * M[:, 1] + h[5]) * ww
        z = np.zeros(len(M))
        Jx = np.stack([M[:, 0] * ww, M[:, 1] * ww, ww, z, z, z, -M[:, 0] * ww * xi, -M[:, 1] * ww * xi], 1)
        Jy = np.stack([z, z, z, M[:, 0] * ww, M[:, 1] * ww, ww, -M[:, 0] * ww * yi, -M[:, 1] * ww * yi], 1)
        return np.concatenate([xi - m[:, 0], yi - m[:, 1]]), np.concatenate([Jx, Jy])
    return compute


# ------------------------------------------------------------------------------------------------ RANSAC driver
@dataclass
class Result:
    ok: bool = False
    model: np.ndarray = None        # best hypothesis (2x3 or 3x3), unrefined
    refined: np.ndarray = None      # what cv2 returns
    inliers: np.ndarray = field(default_factory=lambda: np.zeros(0, np.int64))   # ordered indices, best model
    final: np.ndarray = field(default_factory=lambda: np.zeros(0, np.int64))     # the mask cv2 returns, ordered
    iters: int = 0                  # hypotheses the serial loop evaluated
    err: np.ndarray = None          # float32 error of every point under `model`
    draws: int = 0                  # RNG draws consumed
    hypotheses: list = None         # (subset, model) of every evaluated iteration, when record=True

    @property
    def mask(self):
        """cv2's inlier mask (`final` as booleans)."""
        return None if self.err is None else np.isin(np.arange(len(self.err)), self.final)


def run(prev, cur, kind, max_iters=500, conf=0.99, thresh=3.0, affine_precision="float", refine_iters=10,
        record=False):
    """RANSACPointSetRegistrator::run plus the refinement of cv2.findHomography ("homography") or
    cv2.estimateAffinePartial2D ("affine")."""
    prev, cur = np.asarray(prev, f32).reshape(-1, 2), np.asarray(cur, f32).reshape(-1, 2)
    n = len(prev)
    k = 4 if kind == "homography" else 2
    res = Result(hypotheses=[] if record else None)
    if n < k:
        return res
    thr2 = f32(thresh * thresh)

    def err_of(model):
        if kind == "homography":
            return homography_error(model, prev, cur)
        return affine_error(model, prev, cur, affine_precision)

    if n == k:                  # count == modelPoints: one kernel run, every point an inlier, no refinement
        model = homography_from4(prev, cur) if kind == "homography" else affine_partial_from2(prev, cur)
        if model is None:
            return res
        res.ok, res.model, res.refined = True, model, model
        res.inliers, res.err = np.arange(n), err_of(model)
        res.final = res.inliers
        return res
    rng = CvRng()
    check = None
    if kind == "homography":
        def check(idx):
            return homography_check_subset(prev[idx], cur[idx])
    niters, max_good, best, it = max(max_iters, 1), 0, None, 0
    while it < niters:
        idx = get_subset(n, k, rng, check)
        if idx is None:
            if it == 0:
                return res
            break
        model = homography_from4(prev[idx], cur[idx]) if kind == "homography" else affine_partial_from2(
            prev[idx], cur[idx])
        if record:
            res.hypotheses.append((idx, model))
        if model is not None:
            good = int((err_of(model) <= thr2).sum())
            if good > max(max_good, k - 1):
                best, max_good = model, good
                niters = update_num_iters(conf, (n - good) / n, k, niters)
        it += 1
    res.iters, res.draws = it, rng.draws
    if max_good == 0:
        return res
    res.ok, res.model = True, best
    res.err = err_of(best)
    res.inliers = np.flatnonzero(res.err <= thr2)
    src, dst = prev[res.inliers], cur[res.inliers]
    if kind == "homography":
        H = homography_dlt(src, dst)
        H = best if H is None else H
        h = lm_refine(_homography_cb(src, dst), H.ravel()[:8], 10)
        res.refined = np.append(h, 1.).reshape(3, 3)
        # cv2.findHomography returns the mask of the refined model, over every point
        res.final = np.flatnonzero(homography_error(res.refined, prev, cur) <= thr2)
    else:
        x = np.array([best[0, 0], best[1, 0], best[0, 2], best[1, 2]])
        if refine_iters > 0 and len(res.inliers):
            x = lm_refine(_affine_cb(src, dst), x, refine_iters)
        res.refined = np.array([[x[0], -x[1], x[2]], [x[1], x[0], x[3]]])
        res.final = res.inliers       # estimateAffinePartial2D keeps the mask of the best hypothesis
    return res


# ------------------------------------------------------------------------------------------------ flow.py:215-279
def estimate_bbox(tlbr, A):
    """_estimate_bbox: (rounded box, unrounded box)."""
    a, b, tx, ty = A[0, 0], A[1, 0], A[0, 2], A[1, 2]
    nx, ny = a * tlbr[0] - b * tlbr[1] + tx, b * tlbr[0] + a * tlbr[1] + ty
    scale = math.sqrt(a * a + b * b)
    scale = 1. if scale < 0.9 or scale > 1.1 else scale
    w, h = tlbr[2] - tlbr[0] + 1., tlbr[3] - tlbr[1] + 1.
    raw = np.array([nx, ny, nx + w * scale - 1., ny + h * scale - 1.])
    return np.rint(raw), raw


def flow_homography(prev, cur, status, bg_begin, bg_end, max_iters=500, conf=0.99, thresh=3.0, inlier_thresh=4):
    """Camera motion of Flow.predict: the background matches without the last point (`_get_good_match(..., bg_begin,
    -1)`), findHomography, the inlier-count test.  Returns dict(ok, H, idx (good point indices), res, kp_idx)."""
    idx = np.arange(bg_begin, bg_end - 1)
    idx = idx[np.asarray(status[bg_begin:bg_end - 1]).astype(bool)]
    out = dict(ok=False, H=None, idx=idx, res=None, kp_idx=np.zeros(0, np.int64))
    if len(idx) < 4:
        return out
    res = run(prev[idx], cur[idx], "homography", max_iters, conf, thresh)
    out["res"] = res
    if not res.ok or len(res.final) < inlier_thresh:
        return out
    out.update(ok=True, H=res.refined, kp_idx=idx[res.final])
    return out


def flow_affine_serial(prev, cur, status, begins, tlbrs, frame_size, max_iters=500, conf=0.99, thresh=3.0,
                       inlier_thresh=4, max_pts=None, affine_precision="float"):
    """The per-track loop of Flow.predict (flow.py:234-264), tracks in the given order, each one's predicted box
    painted into the foreground mask before the next track is filtered.  max_pts keeps only the first max_pts
    filtered points of a track (the kernel's per-track capacity).  Returns one dict per track: ok, box, raw (unrounded
    box), m (filtered count), kp_idx (global indices of the inliers, in order), ratio, res."""
    W, H = frame_size
    fg = np.full((H, W), 255, np.uint8)
    out = []
    for t in range(len(tlbrs)):
        b0, b1 = int(begins[t]), int(begins[t + 1])
        idx = np.arange(b0, b1)[np.asarray(status[b0:b1]).astype(bool)]
        p2i = np.rint(cur[idx]).astype(np.int32)
        inside = (p2i[:, 0] >= 0) & (p2i[:, 1] >= 0) & (p2i[:, 0] < W) & (p2i[:, 1] < H)
        idx, p2i = idx[inside], p2i[inside]
        idx = idx[fg[p2i[:, 1], p2i[:, 0]] == 255]
        if max_pts is not None:
            idx = idx[:max_pts]
        r = dict(ok=False, box=None, raw=None, m=len(idx), kp_idx=np.zeros(0, np.int64), ratio=None, res=None)
        out.append(r)
        if len(idx) < 3:
            continue
        res = run(prev[idx], cur[idx], "affine", max_iters, conf, thresh, affine_precision)
        r["res"] = res
        if not res.ok:
            continue
        box, raw = estimate_bbox(np.asarray(tlbrs[t], np.float64), res.refined)
        r["raw"] = raw
        if (np.isnan(box).any() or min(box[2], W - 1) < max(box[0], 0) or min(box[3], H - 1) < max(box[1], 0)
                or len(res.inliers) < inlier_thresh):
            continue
        r.update(ok=True, box=box, kp_idx=idx[res.inliers], ratio=len(res.inliers) / len(idx))
        x0, y0, x1, y1 = (max(int(v), 0) for v in box)
        fg[y0:y1 + 1, x0:x1 + 1] = 0
    return out
