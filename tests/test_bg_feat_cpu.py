"""The index rule of the background mask (csrc/klt_image.cu bg_small_kernel) against cv2.resize INTER_NEAREST, and the
FAST corner bound that sizes Flow's background buffers, on the CPU.

OpenCV's resizeNN samples source index floor(d * (1. / (dsize / ssize))).  The rule floor(d * (ssize / dsize)) gives
the next source row or column wherever the exact product d * ssize / dsize is an integer; the mask then reads one
frame row or column too far and a track box edge there flips a whole background row."""
import numpy as np
import pytest

from fastmot_b200.flow import Flow, fast_corner_bound

cv2 = pytest.importorskip("cv2")

# frame sides of common capture sizes and of the sizes the KLT tests run, at background scales 0.03 .. 1.00
SIDES = (1920, 1080, 1280, 720, 1173, 880, 1366, 768, 1281, 721, 640, 480, 1001, 563, 3840, 2160, 960, 540, 1600, 900,
         2560, 1440, 352, 288, 176, 144, 800, 600, 1024)
PAIRS = sorted({(n, round(s / 100 * n)) for n in SIDES for s in range(3, 101)})


def nearest_rule(n, m):
    """Source index of every output index of a side of n resized to m (the kernel's rule, as OpenCV computes it)."""
    return np.minimum(np.floor(np.arange(m) * (1.0 / (m / n))).astype(np.int64), n - 1)


def ratio_rule(n, m):
    return np.minimum(np.floor(np.arange(m) * (n / m)).astype(np.int64), n - 1)


def cv2_nearest(n, m):
    """The source index cv2.resize(INTER_NEAREST) takes for each of m outputs along a side of n, read from u8 images
    (the mask's type) holding the low and the high byte of the index."""
    idx = np.arange(n)
    planes = [np.tile(((idx >> s) & 255).astype(np.uint8), (2, 1)) for s in (0, 8)]
    lo, hi = (cv2.resize(p, (m, 2), interpolation=cv2.INTER_NEAREST)[0].astype(np.int64) for p in planes)
    return lo + 256 * hi


def test_mask_index_rule_matches_cv2_resize_nearest():
    assert len(PAIRS) > 2500
    differ = 0
    for n, m in PAIRS:
        want = cv2_nearest(n, m)
        np.testing.assert_array_equal(nearest_rule(n, m), want, err_msg=f"{n} -> {m}")
        differ += int((ratio_rule(n, m) != want).sum())
    assert differ > 1000, differ


@pytest.mark.parametrize("n,scale,where", [(720, 0.12, [43]), (1080, 0.07, [57]), (1080, 0.19, [41, 82, 123]),
                                           (1080, 0.38, [41, 82, 123]), (1920, 0.08, [77]), (1366, 0.05, [34])])
def test_ratio_rule_reads_the_next_source_index(n, scale, where):
    m = round(scale * n)
    want, old = cv2_nearest(n, m), ratio_rule(n, m)
    bad = np.nonzero(old != want)[0]
    assert set(where) <= set(bad.tolist()), bad
    np.testing.assert_array_equal(old[bad], want[bad] + 1)


@pytest.mark.parametrize("w,h", [(7, 7), (8, 9), (64, 48), (101, 37), (192, 108)])
def test_fast_corner_bound_holds_on_dense_images(w, h):
    """No image keeps more FAST corners than fast_corner_bound(w, h): noise at threshold 0 and a grid of single bright
    pixels every other row and column (the densest pattern FAST can keep) stay within it."""
    rng = np.random.default_rng(w * h)
    bound = fast_corner_bound(w, h)
    fast = cv2.FastFeatureDetector_create(threshold=0)
    for _ in range(20):
        assert len(fast.detect(rng.integers(0, 256, (h, w), dtype=np.uint8))) <= bound
    grid = np.zeros((h, w), np.uint8)
    grid[3::2, 3::2] = 255
    assert len(fast.detect(grid)) <= bound
    assert fast_corner_bound(6, 100) == fast_corner_bound(100, 6) == 0
    assert fast_corner_bound(7, 7) == 1 and fast_corner_bound(8, 9) == 2


def test_fast_threshold_above_255_depends_on_the_column():
    """cv2's FAST above threshold 255: identical corners (one bright pixel of contrast 100 on a flat image, every other
    column) are found in the first columns and not in the last ones, so there is no result to match; Flow refuses such a
    bg_feat_thresh before it touches the device."""
    w = 74
    img = np.full((12, w), 100, np.uint8)
    for i, x in enumerate(range(3, w - 3)):
        img[4 + 4 * (i % 2), x] = 200
    fast = cv2.FastFeatureDetector_create(threshold=255, nonmaxSuppression=False)
    assert len(fast.detect(img)) == 0
    for t in (44, 99):
        fast.setThreshold(t)
        assert sorted(int(k.pt[0]) for k in fast.detect(img)) == list(range(3, w - 3))
    fast.setThreshold(300)
    cols = sorted(int(k.pt[0]) for k in fast.detect(img))
    assert cols and cols[0] == 3 and cols[-1] < w - 4, cols
    with pytest.raises(ValueError, match="bg_feat_thresh"):
        Flow((640, 480), bg_feat_thresh=300)
