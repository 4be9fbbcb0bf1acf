"""oracle/ransac.py pinned to cv2.findHomography / cv2.estimateAffinePartial2D, called with the reference's arguments
(fastmot/flow.py:223-238: RANSAC, maxIters 500, confidence 0.99, threshold 3), on seeded problems from 3 to 4000
points at 0, 10, 50 and 75 % outliers.  The GPU tests compare the kernels with this restatement, so what is pinned
here is what they check: identical inlier masks, and the refined models."""
import numpy as np
import pytest

from oracle import ransac as R

cv2 = pytest.importorskip("cv2")

OUTLIER_FRACTIONS = (0.0, 0.1, 0.5, 0.75)
CORNERS = np.array([[0, 0, 1], [1919, 0, 1], [0, 1079, 1], [1919, 1079, 1.]])


def _problem(seed, kind):
    rng = np.random.default_rng(seed)
    n = int(rng.choice([3, 4, 5, 8, 20, 60, 300, 1000, 4000])) if seed % 5 else int(rng.integers(3, 4001))
    fo = OUTLIER_FRACTIONS[seed % 4]
    src = rng.uniform([0, 0], [1919, 1079], (n, 2)).astype(np.float32)
    ang, sc = rng.uniform(-0.1, 0.1), rng.uniform(0.85, 1.15)
    A = sc * np.array([[np.cos(ang), -np.sin(ang)], [np.sin(ang), np.cos(ang)]])
    if kind == "homography":
        H = np.eye(3)
        H[:2, :2], H[:2, 2], H[2, :2] = A, rng.uniform(-20, 20, 2), rng.uniform(-2e-5, 2e-5, 2)
        q = np.c_[src, np.ones(n)] @ H.T
        dst = q[:, :2] / q[:, 2:]
    else:
        dst = src @ A.T + rng.uniform(-20, 20, 2)
    dst = (dst + rng.normal(0, rng.uniform(0.05, 1.2), (n, 2))).astype(np.float32)
    out = rng.random(n) < fo
    dst[out] += rng.uniform(-80, 80, (int(out.sum()), 2)).astype(np.float32)
    return src, dst


def _cv2(kind, src, dst, max_iters=500):
    f = cv2.findHomography if kind == "homography" else cv2.estimateAffinePartial2D
    M, mask = f(src, dst, method=cv2.RANSAC, maxIters=max_iters, confidence=0.99)
    return M, (None if mask is None else mask.ravel().astype(bool))


def _map(H, pts):
    q = pts @ np.asarray(H).T
    return q[:, :2] / q[:, 2:]


@pytest.mark.parametrize("kind", ["affine", "homography"])
@pytest.mark.parametrize("seed", range(100))
def test_ransac_oracle_matches_cv2(kind, seed):
    src, dst = _problem(seed, kind)
    got = R.run(src, dst, kind)
    if kind == "homography" and len(src) < 4:
        assert not got.ok            # findHomography refuses fewer than 4 matches; flow.py tests the count first
        return
    want, mask = _cv2(kind, src, dst)
    assert got.ok == (want is not None), (len(src), got.ok)
    if want is None:
        return
    np.testing.assert_array_equal(got.mask, mask)
    if kind == "affine":
        np.testing.assert_allclose(got.refined, want, rtol=1e-6, atol=1e-6 * np.abs(want).max())
    elif len(got.inliers) >= 16:
        # with a handful of matches the 8-parameter least-squares surface is flat and the LM paths of the two
        # solvers (LU here, eigen decomposition in OpenCV) end at different points; the masks above still agree
        assert np.abs(_map(got.refined, CORNERS) - _map(want, CORNERS)).max() < 1e-3


@pytest.mark.parametrize("kind", ["affine", "homography"])
@pytest.mark.parametrize("max_iters", [0, 1, 7, 33])
def test_ransac_oracle_iteration_cap_matches_cv2(kind, max_iters):
    """A small maxIters ends the loop early (0 still runs one hypothesis, like OpenCV's MAX(maxIters, 1))."""
    src, dst = _problem(3, kind)       # 75 % outliers: the adaptive count stays above the cap
    want, mask = _cv2(kind, src, dst, max_iters)
    got = R.run(src, dst, kind, max_iters=max_iters)
    assert got.iters == max(max_iters, 1)
    assert got.ok == (want is not None)
    if want is not None:
        np.testing.assert_array_equal(got.mask, mask)


def test_rng_and_update_num_iters():
    rng = R.CvRng()
    # cv::RNG((uint64)-1): the first draws of the multiply-with-carry stream
    first = [rng.next() for _ in range(3)]
    state = R.U64
    for v in first:
        state = ((state & 0xffffffff) * 4164903690 + (state >> 32)) & R.U64
        assert v == state & 0xffffffff
    assert R.CvRng().uniform(5, 5) == 5
    assert R.update_num_iters(0.99, 0.0, 4, 500) == 0             # every point an inlier: stop at once
    assert R.update_num_iters(0.99, 0.75, 4, 500) == 500          # too many outliers: the cap stands
    assert R.update_num_iters(0.99, 0.5, 2, 500) == 16            # log(0.01) / log(0.75) = 16.0


def test_affine_error_is_float_computed_like_opencv():
    """Affine2DEstimatorCallback::computeError rounds the model to float and forms the residual in float.  Points
    whose squared error lies within one float rounding of 9 are inliers under one formula and outliers under the
    double one; cv2's mask follows the float formula."""
    rng = np.random.default_rng(3)
    n_in, n_probe = 40, 12
    src = rng.uniform(100, 900, (n_in + n_probe, 2)).astype(np.float32)
    c, s = 0.98 * np.cos(0.03), 0.98 * np.sin(0.03)
    dst = (src @ np.array([[c, s], [-s, c]]) + [7.3, -4.1] + rng.normal(0, 0.3, src.shape)).astype(np.float32)
    dst[n_in:] += 3.0
    best = R.run(src, dst, "affine").model
    split = 0
    for i in range(n_in, n_in + n_probe):
        th = rng.uniform(0, 2 * np.pi)
        base = best[:, :2] @ src[i].astype(np.float64) + best[:, 2]
        for k in range(-4000, 4000):
            cand = (base + (3.0 + k * 2e-7) * np.array([np.cos(th), np.sin(th)])).astype(np.float32)[None]
            ef = R.affine_error(best, src[i:i + 1], cand, "float")[0]
            ed = R.affine_error(best, src[i:i + 1], cand, "double")[0]
            if (ef <= 9) != (ed <= 9):
                dst[i] = cand[0]
                split += 1
                break
    assert split >= 4
    fl = R.run(src, dst, "affine", affine_precision="float")
    db = R.run(src, dst, "affine", affine_precision="double")
    np.testing.assert_array_equal(fl.model, db.model)            # the probes move no hypothesis' vote
    assert not np.array_equal(fl.mask, db.mask)
    _, mask = _cv2("affine", src, dst)
    np.testing.assert_array_equal(mask, fl.mask)
    assert not np.array_equal(mask, db.mask)


def test_homography_mask_is_the_refined_models():
    """findHomography returns the inliers of the refined model over every match, not the best hypothesis' inliers:
    with 1 px noise the refined model gains matches the 4-point hypothesis missed."""
    rng = np.random.default_rng(7)
    n = 600
    src = rng.uniform([0, 0], [1919, 1079], (n, 2)).astype(np.float32)
    dst = (src * 1.01 + [4, -3] + rng.normal(0, 1.0, (n, 2))).astype(np.float32)
    dst[:60] += rng.uniform(20, 60, (60, 2)).astype(np.float32)
    want, mask = _cv2("homography", src, dst)
    got = R.run(src, dst, "homography")
    np.testing.assert_array_equal(got.mask, mask)
    best = np.zeros(n, bool)
    best[got.inliers] = True
    assert mask.sum() > best.sum()
    np.testing.assert_array_equal(mask, R.homography_error(want, src, dst) <= 9)


def test_flow_affine_serial_matches_cv2_loop():
    """flow_affine_serial restates flow.py:234-264: filter by status, frame and painted foreground, estimate, predict
    the box, paint it.  Three overlapping tracks, the second's points partly under the first's predicted box."""
    rng = np.random.default_rng(11)
    W, H = 640, 480
    tl = [np.array([100., 100, 199, 199]), np.array([150., 150, 259, 259]), np.array([400., 300, 459, 379])]
    prev, cur, begins = [], [], [0]
    for t in tl:
        p = rng.uniform(t[:2], t[2:], (50, 2)).astype(np.float32)
        c = (p + [3, 2] + rng.normal(0, 0.3, p.shape)).astype(np.float32)
        c[:5] += 30
        prev.append(p), cur.append(c), begins.append(begins[-1] + 50)
    prev, cur = np.concatenate(prev), np.concatenate(cur)
    status = np.ones(len(prev), np.uint8)
    status[::7] = 0
    out = R.flow_affine_serial(prev, cur, status, begins, tl, (W, H))
    fg = np.full((H, W), 255, np.uint8)
    for k, t in enumerate(tl):
        idx = np.arange(begins[k], begins[k + 1])[status[begins[k]:begins[k + 1]] == 1]
        p2i = np.rint(cur[idx]).astype(np.int32)
        idx = idx[fg[p2i[:, 1], p2i[:, 0]] == 255]
        assert out[k]["m"] == len(idx)
        A, mask = _cv2("affine", prev[idx], cur[idx])
        np.testing.assert_array_equal(out[k]["kp_idx"], idx[mask])
        tlp = A @ np.array([t[0], t[1], 1.])
        sc = np.linalg.norm(A[:, 0])
        sc = 1. if sc < 0.9 or sc > 1.1 else sc
        box = np.rint([tlp[0], tlp[1], tlp[0] + (t[2] - t[0] + 1) * sc - 1, tlp[1] + (t[3] - t[1] + 1) * sc - 1])
        np.testing.assert_array_equal(out[k]["box"], box)
        x0, y0, x1, y1 = (max(int(v), 0) for v in box)
        fg[y0:y1 + 1, x0:x1 + 1] = 0
    assert out[1]["m"] < 50 - 50 // 7       # the first track's predicted box covers part of the second's points
