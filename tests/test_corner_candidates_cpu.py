"""The scenes of tests/test_gpu_corner_candidates.py and their corner-candidate counts (no GPU).

A candidate is what cv2.goodFeaturesToTrack sorts before its minimum-distance pass (featureselect.cpp): a local maximum
of the response above qualityLevel times its maximum over the mask, inside the crop's one-pixel border, seen by the
track.  The selection kernel sorts up to 4096 of them in shared memory and more in global memory; these tests pin that
each scene lands where the GPU tests need it, on either side of 4096 and up to about 90 000."""
import numpy as np
import pytest

from fastmot_b200.synth import SyntheticScene, smooth_texture

cv2 = pytest.importorskip("cv2")


def candidate_map(gray, mask=None, bs=3, gs=3, harris=False, quality=0.06):
    """goodFeaturesToTrack candidates of the u8 crop `gray` under `mask` (bool, crop-shaped), as a bool map."""
    e = cv2.cornerHarris(gray, bs, gs, 0.04) if harris else cv2.cornerMinEigenVal(gray, bs, ksize=gs)
    m = np.ones(gray.shape, bool) if mask is None else mask
    t = np.where(e > e[m].max() * quality, e, 0)
    c = (t != 0) & (t == cv2.dilate(t, None)) & m
    c[0, :] = c[-1, :] = c[:, 0] = c[:, -1] = False
    return c


def candidates(gray, mask=None, **kw):
    return int(candidate_map(gray, mask, **kw).sum())


def in_ellipse(c):
    """Candidates of the map `c` inside the ellipse inscribed in the crop (the reference's _ellipse_filter)."""
    h, w = c.shape
    y, x = np.nonzero(c)
    return int((((x - (w - 1) / 2) / (w / 2)) ** 2 + ((y - (h - 1) / 2) / (h / 2)) ** 2 <= 1).sum())


def visible_masks(tlbr, size):
    """Per box, the pixels of its crop no nearer box covers (nearer: lower bottom edge; the scenes have no ties)."""
    W, H = size
    order = np.argsort(-tlbr[:, 3], kind="stable")
    owner = np.full((H, W), -1, np.int64)
    for k in order:
        x0, y0, x1, y1 = np.clip(tlbr[k], 0, [W - 1, H - 1, W - 1, H - 1]).astype(int)
        win = owner[y0:y1 + 1, x0:x1 + 1]
        win[win < 0] = k
    out = []
    for k in range(len(tlbr)):
        x0, y0, x1, y1 = np.clip(tlbr[k], 0, [W - 1, H - 1, W - 1, H - 1]).astype(int)
        out.append(((x0, y0, x1, y1), owner[y0:y1 + 1, x0:x1 + 1] == k))
    return out


def box_candidates(frame, tlbr, **kw):
    gray = cv2.cvtColor(frame, cv2.COLOR_BGR2GRAY)
    H, W = gray.shape
    return [candidates(gray[y0:y1 + 1, x0:x1 + 1], m, **kw) if m.any() else 0
            for (x0, y0, x1, y1), m in visible_masks(tlbr, (W, H))]


def _tlbr(boxes):
    return np.array([(x, y, x + w - 1, y + h - 1) for x, y, w, h in boxes], np.float64)


# ------------------------------------------------------------------------------------------------ scenes
def large_box_scene():
    """1920x1080: a 1000x1000 box of factor-3 texture (about 43 000 candidates), a 640x640 box of factor-6 texture
    (about 8 000) behind three nearer ordinary boxes, and seven more ordinary boxes."""
    rng = np.random.default_rng(31)
    W, H = 1920, 1080
    frame = smooth_texture(rng, H, W, 10)
    boxes = [(30, 40, 1000, 1000), (1220, 20, 640, 640)]
    frame[40:1040, 30:1030] = smooth_texture(rng, 1000, 1000, 3)
    frame[20:660, 1220:1860] = smooth_texture(rng, 640, 640, 6)
    small = [(1250, 500, 80, 170), (1450, 520, 90, 160), (1700, 480, 70, 190), (1100, 760, 56, 96),
             (1200, 800, 50, 90), (1350, 820, 60, 80), (1500, 760, 48, 100), (1600, 900, 52, 88), (1750, 850, 56, 96),
             (1850, 700, 50, 94)]
    for x, y, w, h in small:
        frame[y:y + h, x:x + w] = smooth_texture(rng, h, w, 6)
    return frame, _tlbr(boxes + small)


def cfg_scene(bs, gs, harris):
    """1280x720 as tests/test_gpu_flow_cfg.py's corner scene, with the large box sized to about 4 700 candidates under
    this goodFeaturesToTrack setting (more than 4096, fewer than 4096 inside the box's ellipse, so that maxCorners 0
    with minDistance 1 keeps them all) and eight ordinary boxes beside it."""
    rng = np.random.default_rng(17)
    W, H = 1280, 720
    frame = smooth_texture(rng, H, W, 10)
    fine = smooth_texture(rng, 700, 700, 3)
    g = cv2.cvtColor(fine, cv2.COLOR_BGR2GRAY)
    side = 700
    for _ in range(3):      # the candidate density varies over the texture: refine the side on the crop itself
        side = int(min(700, side * np.sqrt(4700 / candidates(g[:side, :side], bs=bs, gs=gs, harris=harris))))
    boxes = [(10, 10, side, side)]
    frame[10:10 + side, 10:10 + side] = fine[:side, :side]
    for i in range(8):
        x, y = 740 + 75 * (i % 5), 60 + 220 * (i // 5)
        w, h = 56, 96
        frame[y:y + h, x:x + w] = smooth_texture(rng, h, w, 6)
        boxes.append((x, y, w, h))
    return frame, _tlbr(boxes)


# crops of smooth_texture(default_rng(5), 700, 700, 6) in gray with exactly 4095, 4096 and 4097 candidates
BOUNDARY_CROPS = {4095: (437, 440), 4096: (474, 410), 4097: (464, 419)}


def boundary_scene(n_cand):
    """1280x720 with one box showing the top-left (w, h) crop of the boundary texture."""
    w, h = BOUNDARY_CROPS[n_cand]
    tex = smooth_texture(np.random.default_rng(5), 700, 700, 6)
    frame = smooth_texture(np.random.default_rng(7), 720, 1280, 10)
    frame[100:100 + h, 200:200 + w] = tex[:h, :w]
    return frame, _tlbr([(200, 100, w, h)])


def whole_frame_scene():
    """1920x1080 of factor-3 texture, one box over the whole frame (about 90 000 candidates)."""
    frame = smooth_texture(np.random.default_rng(23), 1080, 1920, 3)
    return frame, _tlbr([(0, 0, 1920, 1080)])


class BigObjectScene(SyntheticScene):
    """SyntheticScene with one more object, the nearest: a `side` x `side` box of factor-3 texture at
    (x0 + vx * t, y0 + vy * t), drawn over the others, which are not detected while it hides them whole.  It is the
    last identity."""

    def __init__(self, n_objects=60, seed=41, side=1000, start=(300, 40), vel=(4, 1)):
        super().__init__(n_objects, seed=seed, label=0, dropout_frames=())
        self.big = smooth_texture(np.random.default_rng(seed + 1), side, side, 3)
        self.side, self.start, self.bvel = side, start, vel
        e = np.random.default_rng(seed + 2).normal(size=(1, self.emb.shape[1]))
        self.emb = np.concatenate([self.emb, (e / np.linalg.norm(e)).astype(np.float32)])

    def big_box(self, t):
        return self.start[0] + self.bvel[0] * t, self.start[1] + self.bvel[1] * t

    def frame(self, t):
        img = super().frame(t)
        x, y = self.big_box(t)
        img[y:y + self.side, x:x + self.side] = self.big
        return img

    def detections(self, t, conf=0.9):
        tlbr, labels, confs, ids = super().detections(t, conf)
        x, y = self.big_box(t)
        big = np.array([[x, y, x + self.side - 1, y + self.side - 1]], np.float64)
        seen = ~((tlbr[:, 0] >= big[0, 0]) & (tlbr[:, 1] >= big[0, 1]) & (tlbr[:, 2] <= big[0, 2]) &
                 (tlbr[:, 3] <= big[0, 3]))
        return (np.concatenate([tlbr[seen], big]), np.concatenate([labels[seen], [self.label]]),
                np.concatenate([confs[seen], [conf]]), np.concatenate([ids[seen], [self.n]]))


# ------------------------------------------------------------------------------------------------ tests
def test_large_box_scene_candidates():
    frame, tlbr = large_box_scene()
    c = box_candidates(frame, tlbr)
    assert 40_000 < c[0] < 47_000, c[0]
    assert 4096 < c[1] < 8_000, c[1]          # the 640x640 box loses part of its candidates to the nearer boxes
    assert max(c[2:]) < 4096, c


@pytest.mark.parametrize("harris", [False, True])
@pytest.mark.parametrize("gs", [1, 5, 7])
@pytest.mark.parametrize("bs", [2, 5, 7])
def test_cfg_scene_candidates(bs, gs, harris):
    frame, tlbr = cfg_scene(bs, gs, harris)
    c = box_candidates(frame, tlbr, bs=bs, gs=gs, harris=harris)
    assert 4096 < c[0] < 6_000, c[0]
    assert max(c[1:]) < 4096, c
    x0, y0, x1, y1 = tlbr[0].astype(int)
    gray = cv2.cvtColor(frame, cv2.COLOR_BGR2GRAY)[y0:y1 + 1, x0:x1 + 1]
    assert in_ellipse(candidate_map(gray, bs=bs, gs=gs, harris=harris)) < 3900


@pytest.mark.parametrize("n_cand", sorted(BOUNDARY_CROPS))
def test_boundary_scene_candidates(n_cand):
    w, h = BOUNDARY_CROPS[n_cand]
    tex = cv2.cvtColor(smooth_texture(np.random.default_rng(5), 700, 700, 6), cv2.COLOR_BGR2GRAY)
    assert candidates(tex[:h, :w]) == n_cand
    frame, tlbr = boundary_scene(n_cand)
    assert box_candidates(frame, tlbr) == [n_cand]


def test_whole_frame_candidates():
    frame, tlbr = whole_frame_scene()
    c, = box_candidates(frame, tlbr)
    assert 85_000 < c < 95_000, c


def test_big_object_scene_candidates():
    scene = BigObjectScene()
    for t in (0, 11):
        tlbr, _, _, ids = scene.detections(t)
        assert ids[-1] == scene.n and tlbr[-1, 2] < 1920 and tlbr[-1, 3] < 1080
        c = box_candidates(scene.frame(t), tlbr)
        assert c[-1] > 30_000, (t, c[-1])
