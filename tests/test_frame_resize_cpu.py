"""CPU: the frame-resize restatement (oracle/resize.py) against cv2.resize INTER_LINEAR bit for bit, on BGR frames and
on cv2's decode of NV12 frames, at downscales, upscales, odd and anisotropic size pairs, the exact-2x area path and an
exact 3x (which stays on the generic path)."""
import functools

import numpy as np
import pytest

cv2 = pytest.importorskip("cv2")

from oracle import resize as ors
from oracle.nv12 import bgr_to_nv12

# (capture (w, h), tracking (w, h))
PAIRS = [
    ((1920, 1080), (1280, 720)), ((3840, 2160), (1920, 1080)), ((3840, 2160), (1280, 720)),
    ((1280, 720), (1920, 1080)), ((999, 555), (1920, 1080)), ((640, 480), (1001, 777)),
    ((1921, 1081), (1280, 720)), ((1920, 1080), (1917, 1077)), ((1000, 700), (333, 211)),
    ((1920, 1088), (1920, 1080)), ((1920, 1080), (1280, 1080)), ((1280, 720), (1280, 1080)),
    ((2, 2), (5, 7)), ((7, 5), (2, 2)),
]
IDS = [f"{s[0]}x{s[1]}-{d[0]}x{d[1]}" for s, d in PAIRS]


@functools.lru_cache(maxsize=4)
def _scene(size):
    from fastmot_b200.synth import SyntheticScene
    return SyntheticScene(64, size=size, seed=5, label=0).frame(3)


def _bgr(size, kind):
    if kind == "scene":
        return _scene(size)
    w, h = size
    return np.random.default_rng(w * 7919 + h).integers(0, 256, (h, w, 3), dtype=np.uint8)


def _diff(got, want):
    assert got.shape == want.shape and got.dtype == want.dtype == np.uint8
    return int((got != want).sum())


@pytest.mark.parametrize("kind", ["noise", "scene"])
@pytest.mark.parametrize("src, dst", PAIRS, ids=IDS)
def test_oracle_equals_cv2_resize_bgr(src, dst, kind):
    img = _bgr(src, kind)
    assert _diff(ors.resize_bgr(img, dst), cv2.resize(img, dst)) == 0


# NV12 needs an even capture size; bgr_to_nv12 (cv2's I420) needs at least 4 rows for the scene frame
NV12_CASES = [pytest.param(s, d, k, id=f"{i}-{k}") for (s, d), i in zip(PAIRS, IDS) for k in ("noise", "scene")
              if s[0] % 2 == 0 and s[1] % 2 == 0 and (k == "noise" or s[1] >= 4)]


@pytest.mark.parametrize("src, dst, kind", NV12_CASES)
def test_oracle_equals_cv2_resize_of_nv12_decode(src, dst, kind):
    w, h = src
    if kind == "noise":
        nv = np.random.default_rng(w * 31 + h).integers(0, 256, (3 * h // 2, w), dtype=np.uint8)
    else:
        nv = bgr_to_nv12(_scene(src))
    want = cv2.resize(cv2.cvtColor(nv, cv2.COLOR_YUV2BGR_NV12), dst)
    assert _diff(ors.resize_nv12(nv, dst), want) == 0


def test_exact_3x_takes_the_generic_path_and_2x_the_area_path():
    """At 3840x2160 -> 1280x720 cv2 is not the 3x3 mean: the generic taps take one source column in three with weight
    2048.  At 3840x2160 -> 1920x1080 the generic weights would be 1024 / 1024; the restatement takes the area path and
    matches cv2."""
    img = _bgr((3840, 2160), "noise")
    s = img.astype(np.int64)
    box3 = sum(s[i::3, j::3] for i in range(3) for j in range(3))
    assert _diff(((box3 + 4) // 9).astype(np.uint8), cv2.resize(img, (1280, 720))) > 0
    x0, x1, a0, a1 = ors.taps(1280, 3840, "col")
    assert np.array_equal(x0, 3 * np.arange(1280) + 1) and np.all(a1 == 0)
    half = cv2.resize(img, (1920, 1080))
    i0, i1, w0, w1 = ors.taps(1080, 2160, "row")
    assert np.all(w0 == 1024) and np.all(w1 == 1024)
    assert _diff(ors.resize_bgr(img, (1920, 1080)), half) == 0


def test_upscale_rows_keep_their_fraction_at_the_edges():
    """The row rule clamps indices only: at 720p -> 1080p the first output row blends source row 0 with itself at
    weights 341 / 1707 (fraction kept), which differs from a zeroed fraction on noise; cv2 agrees with the kept one."""
    i0, i1, w0, w1 = ors.taps(1080, 720, "row")
    assert (i0[0], i1[0]) == (0, 0) and w1[0] > 0 and w0[0] + w1[0] == 2048
    img = _bgr((1280, 720), "noise")
    want = cv2.resize(img, (1920, 1080))
    got = ors.resize_bgr(img, (1920, 1080))
    assert _diff(got, want) == 0
    # the column rule applied to rows (a zeroed fraction at the edges) is off by 1 LSB on the first and last rows
    y0, y1, b0, b1 = ors.taps(1080, 720, "col")
    x0, x1, a0, a1 = ors.taps(1920, 1280, "col")
    s = img.astype(np.int64)
    h = s[:, x0] * a0[:, None] + s[:, x1] * a1[:, None]
    zeroed = ((((b0[:, None, None] * (h[y0] >> 4)) >> 16) + ((b1[:, None, None] * (h[y1] >> 4)) >> 16) + 2)
              >> 2).astype(np.uint8)
    bad = np.nonzero((zeroed != want).any(axis=(1, 2)))[0]
    assert len(bad) > 0 and set(bad.tolist()) <= {0, 1079}
