"""CPU: the KLT stage at other frame sizes, optical-flow scales and goodFeaturesToTrack settings.

* OracleTracker (OpenCV underneath) reproduces tests/golden/seq_flow_cfg.npz, written from the unmodified reference by
  oracle/flow_cfg_goldens.py: an odd-sized camera at the default flow_cfg, an anisotropic scale with blockSize 5
  and no corner limit, full scale with the Harris response and gradient aperture 5.
* The integer restatement of the INTER_LINEAR resize that csrc/klt_image.cu's resize_linear_kernel computes is
  bit-exact against cv2.resize, and the float64 restatement of the corner response that csrc/klt_feat.cu's
  gftt_response_kernel computes matches cv2.cornerMinEigenVal / cv2.cornerHarris.
"""
import itertools
import os

import numpy as np
import pytest

from conftest import GOLDEN
from oracle.flow_cfg_goldens import FLOW_CFG_CASES, flow_cfg_namespace

cv2 = pytest.importorskip("cv2")


def flow_case_cfg(i):
    """default_tracker_cfg() with the flow_cfg of FLOW_CFG_CASES[i]."""
    from oracle.run import default_tracker_cfg
    cfg = default_tracker_cfg()
    _, _, _, flow_over, feat_over = FLOW_CFG_CASES[i]
    cfg['flow_cfg'] = flow_cfg_namespace(cfg['flow_cfg'], flow_over, feat_over)
    return cfg


@pytest.fixture(scope="module")
def golden():
    return np.load(os.path.join(GOLDEN, "seq_flow_cfg.npz"))


@pytest.mark.parametrize("i", range(len(FLOW_CFG_CASES)), ids=[c[0] for c in FLOW_CFG_CASES])
def test_oracle_tracker_reproduces_flow_cfg_golden(i, golden):
    from fastmot_b200.synth import SyntheticScene
    from oracle.tracker import OracleTracker
    name, scene_kw, n_frames, _, _ = FLOW_CFG_CASES[i]
    assert str(golden[f'c{i}_name']) == name
    scene = SyntheticScene(**scene_kw)
    trk = OracleTracker(scene.size, 'cosine', **flow_case_cfg(i))
    trk.reset(1 / 30.)
    for t in range(n_frames):
        frame = scene.frame(t)
        if t == 0:
            tlbr, labels, conf, ids = scene.detections(0)
            trk.init(frame, tlbr, labels)
        else:
            trk.compute_flow(frame)
            assert trk.homography is not None, t
            np.testing.assert_array_equal(trk.homography, golden[f'c{i}_H_{t}'])
            assert list(trk.klt_bboxes) == golden[f'c{i}_klt_ids_{t}'].tolist(), t
            got = np.array([trk.klt_bboxes[k] for k in trk.klt_bboxes], np.float64).reshape(-1, 4)
            np.testing.assert_array_equal(got, golden[f'c{i}_klt_tlbr_{t}'])
            trk.apply_kalman()
            if t % 5 == 0:
                tlbr, labels, conf, ids = scene.detections(t)
                trk.update(t, tlbr, labels, conf, scene.embeddings(ids, t))
        vis = trk.visible()
        assert [k for k, _ in vis] == golden[f'c{i}_vis_ids_{t}'].tolist(), t
        np.testing.assert_array_equal(np.array([b for _, b in vis]).reshape(-1, 4), golden[f'c{i}_vis_tlbr_{t}'])
    assert len(vis) >= 40


# ------------------------------------------------------------------------------------------------ resize
def resize_linear(gray, sw, sh):
    """cv2.resize(gray, (sw, sh)) INTER_LINEAR for u8 at a downscale, as resize_linear_kernel computes it: scale
    1 / (dsize / ssize) in double, source coordinate in float, 11-bit coefficients rounded half to even, the far edge
    clamped with a zero weight, and the vertical pass of OpenCV's VResizeLinearVec_32s8u."""
    H, W = gray.shape

    def coefs(d, s):
        scale = 1.0 / (d / s)
        f = ((np.arange(d) + 0.5) * scale - 0.5).astype(np.float32)
        i = np.floor(f).astype(np.int64)
        f = (f - i).astype(np.float32)
        lo = i < 0
        f[lo], i[lo] = 0, 0
        hi = i >= s - 1
        f[hi], i[hi] = 0, s - 1
        c0 = np.rint((np.float32(1) - f) * np.float32(2048)).astype(np.int64)
        c1 = np.rint(f * np.float32(2048)).astype(np.int64)
        return i, np.minimum(i + 1, s - 1), c0, c1

    x0, x1, a0, a1 = coefs(sw, W)
    y0, y1, b0, b1 = coefs(sh, H)
    g = gray.astype(np.int64)
    h0 = g[y0][:, x0] * a0 + g[y0][:, x1] * a1
    h1 = g[y1][:, x0] * a0 + g[y1][:, x1] * a1
    return ((((b0[:, None] * (h0 >> 4)) >> 16) + ((b1[:, None] * (h1 >> 4)) >> 16) + 2) >> 2).astype(np.uint8)


RESIZE_SIZES = [(1920, 1080), (1173, 880), (1545, 1080), (1281, 721), (640, 480)]
RESIZE_SCALES = [(0.1, 0.1), (0.25, 0.25), (0.33, 0.5), (0.4, 0.6), (0.5, 0.5), (0.75, 0.75), (0.9, 0.2), (1.0, 1.0)]


def test_resize_restatement_bit_exact_against_cv2():
    rng = np.random.default_rng(0)
    checked = 0
    for (W, H), (sx, sy) in itertools.product(RESIZE_SIZES, RESIZE_SCALES):
        sw, sh = round(sx * W), round(sy * H)
        if 2 * sw == W and 2 * sh == H:
            continue            # cv2.resize takes its 2x2-mean path there (fm_gray_half, pinned in test_gpu_klt.py)
        noise = rng.integers(0, 256, (H, W), dtype=np.uint8)
        for img in (noise, cv2.GaussianBlur(noise, (0, 0), 5)):
            np.testing.assert_array_equal(resize_linear(img, sw, sh), cv2.resize(img, (sw, sh)),
                                          err_msg=f"{W}x{H} -> {sw}x{sh}")
            checked += 1
    assert checked >= 70


# ------------------------------------------------------------------------------------------------ corner response
SOBEL_SMOOTH = {1: [1], 3: [1, 2, 1], 5: [1, 4, 6, 4, 1], 7: [1, 6, 15, 20, 15, 6, 1]}
SOBEL_DERIV = {1: [-1, 0, 1], 3: [-1, 0, 1], 5: [-1, -2, 0, 2, 1], 7: [-1, -4, -5, 0, 5, 4, 1]}


def _reflect101(n, lo, hi):
    """Indices of [-lo, n + hi) folded into [0, n) with BORDER_REFLECT_101."""
    idx = np.arange(-lo, n + hi)
    if n == 1:
        return np.zeros_like(idx)
    while (idx < 0).any() or (idx >= n).any():
        idx = np.where(idx < 0, -idx, idx)
        idx = np.where(idx >= n, 2 * n - 2 - idx, idx)
    return idx


def _filter1d(img, taps, axis):
    r = len(taps) // 2
    src = np.take(img, _reflect101(img.shape[axis], r, r), axis=axis)
    out = np.zeros(img.shape, np.float64)
    for j, c in enumerate(taps):
        out += c * np.take(src, np.arange(j, j + img.shape[axis]), axis=axis)
    return out


def structure_tensor(img, block_size, ksize):
    """float64 pass 1 + box sums of gftt_response_kernel: Sobel of aperture ksize (reflect-101) scaled by
    1 / (2^(ksize-1) * block * 255), the gradient products summed over the unnormalised block window anchored at
    block // 2 (reflect-101).  Returns (sum Dx^2, sum Dx*Dy, sum Dy^2)."""
    g = img.astype(np.float64)
    scale = 1.0 / ((1 << (ksize - 1)) * block_size * 255.0)
    dx = _filter1d(_filter1d(g, SOBEL_DERIV[ksize], 1), SOBEL_SMOOTH[ksize], 0) * scale
    dy = _filter1d(_filter1d(g, SOBEL_SMOOTH[ksize], 1), SOBEL_DERIV[ksize], 0) * scale
    anchor = block_size // 2
    H, W = img.shape
    rows = _reflect101(H, anchor, block_size - 1 - anchor)
    cols = _reflect101(W, anchor, block_size - 1 - anchor)

    def box(p):
        p = p[rows][:, cols]
        return sum(p[j:j + H, i:i + W] for j in range(block_size) for i in range(block_size))

    return box(dx * dx), box(dx * dy), box(dy * dy)


def corner_response(img, block_size, ksize, harris_k=None):
    """The minimum eigenvalue of the structure tensor or, with harris_k, a*c - b^2 - k*(a+c)^2."""
    a, b, c = structure_tensor(img, block_size, ksize)
    if harris_k is not None:
        return a * c - b * b - harris_k * (a + c) ** 2
    a, c = a * 0.5, c * 0.5
    return (a + c) - np.sqrt((a - c) ** 2 + b * b)


@pytest.mark.parametrize("block_size", [1, 2, 3, 4, 5, 7])
@pytest.mark.parametrize("ksize", [1, 3, 5, 7])
def test_corner_response_restatement_against_cv2(block_size, ksize):
    from fastmot_b200.synth import SyntheticScene
    scene = SyntheticScene(60, seed=6)
    gray = cv2.cvtColor(scene.frame(2), cv2.COLOR_BGR2GRAY)
    tlbr = scene.detections(2)[0].astype(int)
    # two object boxes and one window over several objects and the background
    for (x0, y0, x1, y1) in [tlbr[0], tlbr[7], (tlbr[20][0], tlbr[20][1], tlbr[20][0] + 150, tlbr[20][1] + 120)]:
        crop = np.ascontiguousarray(gray[y0:y1 + 1, x0:x1 + 1])
        # errors are float32 rounding of the tensor entries: bound them by its largest trace (the minimum eigenvalue
        # at blockSize 1 is identically zero and OpenCV returns rounding noise there)
        a, _, c = structure_tensor(crop, block_size, ksize)
        tr = (a + c).max()
        assert tr > 0
        want = cv2.cornerMinEigenVal(crop, block_size, ksize=ksize).astype(np.float64)
        got = corner_response(crop, block_size, ksize)
        assert np.abs(got - want).max() <= 1e-6 * tr, (x0, np.abs(got - want).max() / tr)
        want = cv2.cornerHarris(crop, block_size, ksize, 0.04).astype(np.float64)
        got = corner_response(crop, block_size, ksize, harris_k=0.04)
        assert np.abs(got - want).max() <= 1e-6 * tr * tr, (x0, np.abs(got - want).max() / tr ** 2)
        if block_size > 1:
            assert np.abs(got - want).max() <= 1e-5 * np.abs(want).max()


def test_flow_rejects_what_opencv_rejects():
    from fastmot_b200.flow import Flow
    from types import SimpleNamespace as NS
    with pytest.raises(ValueError, match="gradientSize"):
        Flow((1173, 880), obj_feat_params=NS(gradientSize=4))
    with pytest.raises(ValueError, match="blockSize"):
        Flow((1173, 880), obj_feat_params=NS(blockSize=0))
    with pytest.raises(ValueError, match="empty optical-flow image"):
        Flow((3, 880), opt_flow_scale_factor=(0.1, 0.5))
    with pytest.raises(TypeError, match="minDistance"):
        Flow((1173, 880), obj_feat_params=NS(minDistance=3))
