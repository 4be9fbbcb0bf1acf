"""GPU parity of the KLT background stage of Flow.predict (fastmot/flow.py:186-200) against OpenCV 4.13, bit for bit
(DESIGN.md a11): the background image and mask (fm_bg_small) against cv2.resize INTER_LINEAR / INTER_NEAREST, the
corners (fm_fast_detect) against cv2.FastFeatureDetector, at every frame size, background scale, FAST threshold, mask
and image size below, and Flow end to end against the oracle at background scales whose mask rows the old sampling
rule got wrong."""
import numpy as np
import pytest
import torch

from test_bg_feat_cpu import nearest_rule, ratio_rule

cv2 = pytest.importorskip("cv2")
pytestmark = pytest.mark.gpu

NO_OWNER = 0x7fffffff


# ------------------------------------------------------------------------------------------------ device calls
def gpu_bg_small(gray, owner, bw, bh):
    """fm_bg_small on a host gray image and owner map: (background image, mask)."""
    from fastmot_b200 import _lib
    from fastmot_b200.devmem import ptr, stream_ptr
    lib = _lib.load()
    h, w = gray.shape
    g, o = torch.as_tensor(gray).cuda(), torch.as_tensor(owner).cuda()
    bg = torch.full((bh, bw), 7, dtype=torch.uint8, device="cuda")
    mask = torch.full((bh, bw), 7, dtype=torch.uint8, device="cuda")
    _lib.check(lib.fm_bg_small(ptr(g), ptr(o), w, h, ptr(bg), ptr(mask), bw, bh, stream_ptr()), "fm_bg_small")
    torch.cuda.synchronize()
    return bg.cpu().numpy(), mask.cpu().numpy()


def gpu_fast(img, mask, threshold, unscale=(1.0, 1.0), max_pts=None):
    """fm_fast_detect on a host image and mask: (points (N, 2) f32, score image)."""
    from fastmot_b200 import _lib
    from fastmot_b200.flow import fast_corner_bound
    from fastmot_b200.devmem import ptr, stream_ptr
    lib = _lib.load()
    h, w = img.shape
    max_pts = max_pts or max(fast_corner_bound(w, h), 1)
    im, mk = torch.as_tensor(img).cuda(), torch.as_tensor(mask).cuda()
    score = torch.full((h, w), 7, dtype=torch.uint8, device="cuda")
    pts = torch.full((max_pts + 1, 2), -1.0, dtype=torch.float32, device="cuda")
    cnt = torch.full((1,), -1, dtype=torch.int32, device="cuda")
    _lib.check(lib.fm_fast_detect(ptr(im), ptr(mk), w, h, int(threshold), float(unscale[0]), float(unscale[1]),
                                  ptr(score), ptr(pts), ptr(cnt), max_pts, stream_ptr()), "fm_fast_detect")
    torch.cuda.synchronize()
    n = int(cnt.item())
    assert 0 <= n <= max_pts
    assert (pts[max_pts] == -1).all()                 # nothing written past max_pts
    return pts[:n].cpu().numpy(), score.cpu().numpy()


# ------------------------------------------------------------------------------------------------ A. fm_bg_small
SIZES = [(1920, 1080), (1280, 720), (1173, 880), (1366, 768), (1281, 721), (640, 480), (1001, 563)]
SCALES = [(0.05, 0.05), (0.07, 0.07), (0.1, 0.1), (0.12, 0.12), (0.15, 0.15), (0.19, 0.19), (0.25, 0.25),
          (0.38, 0.38), (0.5, 0.5), (1.0, 1.0), (0.9, 0.2), "one"]


def bg_size(size, scale):
    """Background image size of Flow at this frame size and scale ("one": one column wide)."""
    W, H = size
    if scale == "one":
        scale = (0.6 / W, 0.1)
    return round(scale[0] * W), round(scale[1] * H)


def flipped(n, m):
    """(output index, the source index cv2 samples, the one the w / bw rule sampled) where the two differ."""
    new, old = nearest_rule(n, m), ratio_rule(n, m)
    return [(d, int(new[d]), int(old[d])) for d in np.nonzero(new != old)[0]]


def adversarial_owner(size, bw, bh):
    """An owner map with a box edge between the two source rows (columns) of every flipped mask row (column): the box
    covers the row cv2 samples and not the other one, so a mask read from the wrong row flips that row."""
    W, H = size
    owner = np.full((H, W), NO_OWNER, np.int32)
    k = 0
    for _, a, b in flipped(H, bh):
        lo, hi = sorted((a, b))
        owner[max(lo - 2, 0):lo + 1, k % 3:W // 2 + k % 3] = k
        k += 1
    for _, a, b in flipped(W, bw):
        lo, hi = sorted((a, b))
        owner[k % 5:H // 2, max(lo - 2, 0):lo + 1] = k
        k += 1
    return owner


def random_owner(size, rng, n=40):
    W, H = size
    owner = np.full((H, W), NO_OWNER, np.int32)
    for k in range(n):
        x0, y0 = rng.integers(0, W), rng.integers(0, H)
        owner[y0:y0 + rng.integers(1, H // 3 + 2), x0:x0 + rng.integers(1, W // 3 + 2)] = k
    return owner


def test_parameter_set_covers_the_flipped_indices():
    """The adversarial maps only test something at sizes and scales where the two floor rules differ: the set must
    keep such cases, among them 1280x720 at 0.12 (row 43) and 1920x1080 at 0.38 (rows 41, 82, 123)."""
    cases = {(size, scale): flipped(size[1], bg_size(size, scale)[1]) + flipped(size[0], bg_size(size, scale)[0])
             for size in SIZES for scale in SCALES}
    assert [d for d, _, _ in cases[(1280, 720), (0.12, 0.12)]] == [43]
    assert {41, 82, 123} <= {d for d, _, _ in cases[(1920, 1080), (0.38, 0.38)]}
    assert [d for d, _, _ in cases[(1366, 768), (0.05, 0.05)]] == [34]
    assert sum(bool(v) for v in cases.values()) >= 8, sum(bool(v) for v in cases.values())


@pytest.mark.parametrize("scale", SCALES, ids=[str(s) for s in SCALES])
@pytest.mark.parametrize("size", SIZES, ids=[f"{w}x{h}" for w, h in SIZES])
def test_bg_small_vs_cv2_resize(size, scale):
    """Background image = cv2.resize(gray, (bw, bh)) (INTER_LINEAR; cv2's 2x2 mean at 0.5, a copy at 1.0) and mask =
    cv2.resize(fg, (bw, bh), INTER_NEAREST) for random boxes and for the adversarial box edges."""
    W, H = size
    bw, bh = bg_size(size, scale)
    rng = np.random.default_rng(W * 7 + H)
    gray = rng.integers(0, 256, (H, W), dtype=np.uint8)
    gray[: H // 2] = cv2.GaussianBlur(gray[: H // 2], (5, 5), 1.5)       # smooth and noisy halves
    for owner in (random_owner(size, rng), adversarial_owner(size, bw, bh)):
        fg = np.where(owner == NO_OWNER, 255, 0).astype(np.uint8)
        want_mask = cv2.resize(fg, (bw, bh), interpolation=cv2.INTER_NEAREST)
        bg, mask = gpu_bg_small(gray, owner, bw, bh)
        np.testing.assert_array_equal(bg, cv2.resize(gray, (bw, bh)), err_msg=f"{size} {scale} image")
        np.testing.assert_array_equal(mask, want_mask, err_msg=f"{size} {scale} mask")
    if flipped(H, bh) or flipped(W, bw):
        # the adversarial map does catch the old rule here
        old = fg[ratio_rule(H, bh)][:, ratio_rule(W, bw)]
        assert not np.array_equal(old, want_mask)


# ------------------------------------------------------------------------------------------------ B. fm_fast_detect
THRESHOLDS = [0, 1, 10, 37, 128, 254, 255]
FAST_SIZES = [(6, 20), (20, 6), (5, 5), (7, 7), (8, 9), (101, 37), (192, 108), (512, 256), (363, 362), (576, 324),
              (730, 410), (1920, 1080)]


CIRCLE = [(0, 3), (1, 3), (2, 2), (3, 1), (3, 0), (3, -1), (2, -2), (1, -3), (0, -3), (-1, -3), (-2, -2), (-3, -1),
          (-3, 0), (-3, 1), (-2, 2), (-1, 3)]      # (dx, dy) of FAST's Bresenham circle, index 0 .. 15


def cv2_fast(img, mask, t, unscale=(1.0, 1.0)):
    kp = cv2.FastFeatureDetector_create(threshold=t).detect(img, mask=mask)
    return np.asarray(cv2.KeyPoint_convert(kp), np.float32).reshape(-1, 2) * np.asarray(unscale, np.float32)


def cv2_fast_scores(img, t):
    """The score image of fast_score_kernel: 0 except at the corners cv2 detects without non-max suppression, where it
    is OpenCV's cornerScore, restated: the contrast of the best 9-pixel arc, darker or brighter, minus 1.  cv2 leaves
    the response 0 without suppression, so the restatement is checked against the response of every corner cv2 keeps
    with suppression."""
    kp = cv2.FastFeatureDetector_create(threshold=t, nonmaxSuppression=False).detect(img)
    score = np.zeros(img.shape, np.uint8)
    if not kp:
        return score
    xy = np.rint(np.asarray(cv2.KeyPoint_convert(kp))).astype(np.int64)
    v = img[xy[:, 1], xy[:, 0]].astype(np.int64)
    d = np.stack([v - img[xy[:, 1] + dy, xy[:, 0] + dx] for dx, dy in CIRCLE], 1)
    d = np.concatenate([d, d[:, :8]], 1)
    arcs = np.stack([d[:, s:s + 9] for s in range(16)], 1)             # (corners, 16 arcs, 9 pixels)
    best = np.maximum(arcs.min(2).max(1), (-arcs).min(2).max(1))
    score[xy[:, 1], xy[:, 0]] = best - 1
    kept = cv2.FastFeatureDetector_create(threshold=t).detect(img)
    if kept:
        kxy = np.rint(np.asarray(cv2.KeyPoint_convert(kept))).astype(np.int64)
        np.testing.assert_array_equal(score[kxy[:, 1], kxy[:, 0]], [k.response for k in kept])
    return score


def fast_image(kind, size, seed):
    w, h = size
    rng = np.random.default_rng(seed)
    if kind == "uniform":
        return rng.integers(0, 256, (h, w), dtype=np.uint8)
    if kind == "blurred":
        return cv2.GaussianBlur(rng.integers(0, 256, (h, w), dtype=np.uint8), (5, 5), 1.2)
    from fastmot_b200.synth import SyntheticScene
    W, H = max(w, 64), max(h, 64)
    gray = cv2.cvtColor(SyntheticScene(40, size=(W, H), seed=seed).frame(3), cv2.COLOR_BGR2GRAY)
    return np.ascontiguousarray(gray[:h, :w])


def fast_masks(size, seed):
    w, h = size
    rng = np.random.default_rng(seed + 1)
    blocks = np.kron(rng.integers(0, 2, ((h + 7) // 8, (w + 7) // 8)), np.ones((8, 8), np.int64))[:h, :w]
    return {"all255": np.full((h, w), 255, np.uint8), "all0": np.zeros((h, w), np.uint8),
            "random": np.where((blocks > 0) | (rng.random((h, w)) < 0.1), 255, 0).astype(np.uint8)}


@pytest.mark.parametrize("kind", ["uniform", "blurred", "scene"])
@pytest.mark.parametrize("size", FAST_SIZES, ids=[f"{w}x{h}" for w, h in FAST_SIZES])
def test_fast_points_vs_cv2(size, kind):
    """Same count, same row-major order, same unscaled coordinates as cv2.FastFeatureDetector + _unscale_pts, at
    every threshold 0 .. 255 and mask; sizes with no interior, not a multiple of 32 pixels, and either side of 131 072."""
    img = fast_image(kind, size, seed=size[0] + size[1])
    unscale = (float(np.float32(1) / np.float32(0.38)), float(np.float32(1) / np.float32(0.1)))
    for name, mask in fast_masks(size, size[0]).items():
        for t in THRESHOLDS:
            want = cv2_fast(img, mask, t, unscale)
            got, _ = gpu_fast(img, mask, t, unscale)
            assert got.shape == want.shape, (size, kind, name, t, got.shape, want.shape)
            np.testing.assert_array_equal(got, want, err_msg=f"{size} {kind} {name} t={t}")


@pytest.mark.parametrize("kind", ["uniform", "blurred", "scene"])
@pytest.mark.parametrize("size", [(7, 7), (101, 37), (192, 108), (363, 362), (730, 410)],
                         ids=lambda s: f"{s[0]}x{s[1]}")
def test_fast_scores_vs_cv2_response(size, kind):
    """fast_score_kernel: the score of every corner equals cv2's response (best arc minus 1, nonmaxSuppression=False),
    and every other pixel scores 0."""
    img = fast_image(kind, size, seed=3 * size[0] + size[1])
    ones = np.full(img.shape, 255, np.uint8)
    for t in THRESHOLDS:
        _, score = gpu_fast(img, ones, t)
        np.testing.assert_array_equal(score, cv2_fast_scores(img, t), err_msg=f"{size} {kind} t={t}")


def hand_built(t):
    """A 96x64 image of flat 100 with hand-placed FAST cases for threshold t; returns (image, {name: (x, y)})."""
    img = np.full((64, 96), 100, np.uint8)
    at = {}

    def arc(x, y, start, length, delta):
        for k in range(start, start + length):
            dx, dy = CIRCLE[k % 16]
            img[y + dy, x + dx] = np.clip(100 + delta, 0, 255)

    c = min(t, 150)
    # arcs of 8 and 9, darker and brighter, at contrast t and t + 1
    for j, (length, delta) in enumerate([(9, c + 1), (9, c), (8, c + 1), (9, -(c + 1)), (9, -c), (8, -(c + 1))]):
        x, y = 8 + 10 * j, 8
        arc(x, y, 3, length, delta)
        at[f"arc{length}_{delta}"] = (x, y)
    # arcs that wrap from circle index 15 to 0
    arc(8, 20, 12, 9, c + 1); at["wrap_bright"] = (8, 20)
    arc(18, 20, 10, 10, -(c + 1)); at["wrap_dark"] = (18, 20)
    # a brighter arc of 9 and a darker arc of 7 around one pixel, then arcs of 8 and 8
    arc(30, 20, 0, 9, 60); arc(30, 20, 9, 7, -90); at["both_9_7"] = (30, 20)
    arc(42, 20, 0, 8, 60); arc(42, 20, 8, 8, -90); at["both_8_8"] = (42, 20)
    # a 9-pixel arc of contrast 60: cornerScore 59 when t < 60
    arc(54, 20, 5, 9, -60); at["arc9_60"] = (54, 20)
    # equal-score neighbours (two bright pixels side by side: cv2 keeps neither) and unequal ones
    img[32, 8] = img[32, 9] = 200; at["equal_pair"] = (8, 32)
    img[32, 20] = 200; img[32, 21] = 180; at["strong"] = (20, 32); at["weak"] = (21, 32)
    img[44, 20] = 200; img[45, 21] = 180; at["strong_diag"] = (20, 44); at["weak_diag"] = (21, 45)
    img[32, 34] = 200; at["single"] = (34, 32)
    # corners on the first and last rows / columns FAST examines (3 and w-4 / h-4), and just outside them
    for x, y in [(3, 56), (92, 40), (60, 3), (70, 60), (2, 48), (93, 28), (80, 2), (86, 61)]:
        img[y, x] = 230
        at[f"edge_{x}_{y}"] = (x, y)
    return img, at


@pytest.mark.parametrize("t", THRESHOLDS)
def test_fast_hand_built_corners(t):
    """Arcs of 8 and 9 at contrast t and t+1, wrapping arcs, a brighter and a darker arc around one pixel, equal and
    unequal neighbours, corners on the border rows / columns; then a mask 0 on the stronger of two neighbours: cv2 runs
    NMS before the mask, so the masked corner still suppresses the weaker one."""
    img, at = hand_built(t)
    ones = np.full(img.shape, 255, np.uint8)
    want = cv2_fast(img, ones, t)
    got, score = gpu_fast(img, ones, t)
    np.testing.assert_array_equal(got, want)
    np.testing.assert_array_equal(score, cv2_fast_scores(img, t))
    kept = {tuple(p) for p in want.astype(int).tolist()}
    if t <= 60:
        assert at["single"] in kept and at["strong"] in kept and at["weak"] not in kept
        assert at["equal_pair"] not in kept and (9, 32) not in kept
        assert at["edge_3_56"] in kept and at["edge_92_40"] in kept and at["edge_60_3"] in kept
        assert at["edge_2_48"] not in kept and at["edge_93_28"] not in kept and at["edge_80_2"] not in kept
    if t < 60:
        assert score[at["arc9_60"][::-1]] == 59
    if 0 < t <= 150:
        assert at[f"arc9_{t + 1}"] in kept and at[f"arc9_{t}"] not in kept and at[f"arc8_{t + 1}"] not in kept
        assert at["wrap_bright"] in kept
    if 0 < t < 100:                                 # darker arcs reach contrast t + 1 below 100 (flat image = 100)
        assert at[f"arc9_{-(t + 1)}"] in kept and at[f"arc9_{-t}"] not in kept and at["wrap_dark"] in kept
    mask = ones.copy()
    for name in ("strong", "strong_diag"):
        x, y = at[name]
        mask[y, x] = 0
    want = cv2_fast(img, mask, t)
    got, _ = gpu_fast(img, mask, t)
    np.testing.assert_array_equal(got, want)
    kept = {tuple(p) for p in want.astype(int).tolist()}
    assert at["weak"] not in kept and at["weak_diag"] not in kept and at["strong"] not in kept


def test_fast_threshold_above_255_is_refused():
    """cv2's FAST gives no single answer above threshold 255 (tests/test_bg_feat_cpu.py): fm_fast_detect refuses it
    rather than return corners no OpenCV call reproduces."""
    from fastmot_b200._lib import FastMOTLibError
    img = fast_image("uniform", (101, 37), 1)
    ones = np.full(img.shape, 255, np.uint8)
    for t in (256, 300, -1):
        with pytest.raises(FastMOTLibError, match="threshold"):
            gpu_fast(img, ones, t)
    got, _ = gpu_fast(img, ones, 255)
    np.testing.assert_array_equal(got, cv2_fast(img, ones, 255))


# ------------------------------------------------------------------------------------------------ C. capacity
def test_fast_never_clips_and_caps_at_max_pts():
    """Flow sizes its background buffers to the most corners the image can keep, whatever max_bg_points says; the
    kernel itself writes at most max_pts points."""
    from fastmot_b200.flow import Flow, fast_corner_bound
    f = Flow((1920, 1080), bg_feat_scale_factor=(1.0, 1.0), max_bg_points=16, scratch_floats=1 << 10)
    assert f.max_bg == fast_corner_bound(1920, 1080) and f.bg_pts.shape[0] == f.max_bg
    assert Flow((1920, 1080), max_bg_points=1 << 16, scratch_floats=1 << 10).max_bg == 1 << 16
    img = fast_image("uniform", (363, 362), 5)
    ones = np.full(img.shape, 255, np.uint8)
    want = cv2_fast(img, ones, 0)
    assert len(want) > 10000
    got, _ = gpu_fast(img, ones, 0)
    np.testing.assert_array_equal(got, want)
    got, _ = gpu_fast(img, ones, 0, max_pts=1000)
    np.testing.assert_array_equal(got, want[:1000])


def _dets(tlbr, labels, conf):
    dt = np.dtype([('tlbr', float, 4), ('label', int), ('conf', float)], align=True)
    arr = np.zeros(len(tlbr), dt)
    arr['tlbr'], arr['label'], arr['conf'] = tlbr, labels, conf
    return arr.view(np.recarray)


@pytest.mark.parametrize("use_runner", [True, False], ids=["runner", "calls"])
def test_max_points_overflow_raises(monkeypatch, use_runner):
    """More track keypoints and background corners than max_points raise a MemoryError naming max_points (the
    overflow flag travels with the flow status read-back), on both enqueue paths; it never returns a short list."""
    from fastmot_b200 import MultiTracker
    from fastmot_b200.flow import Flow
    from fastmot_b200.synth import SyntheticScene
    from oracle.run import default_tracker_cfg
    monkeypatch.setattr(Flow, "USE_RUNNER", use_runner)
    scene = SyntheticScene(40, seed=8)
    cfg = default_tracker_cfg()
    cfg['flow_cfg'].max_points = 300
    trk = MultiTracker(scene.size, 'cosine', **cfg)
    trk.reset(1 / 30)
    tl, lb, cf, _ = scene.detections(0)
    trk.init(scene.frame(0), _dets(tl, lb, cf))
    trk.compute_flow(scene.frame(1))
    with pytest.raises(MemoryError, match="max_points=300"):
        trk.apply_kalman()
    f = Flow(scene.size, **vars(cfg['flow_cfg']))
    f.bind_pool(trk.pool)
    f.init(scene.frame(0))
    with pytest.raises(MemoryError, match="max_points=300"):
        f.predict(scene.frame(1), [t for t in trk.tracks.values()])


# ------------------------------------------------------------------------------------------------ D. Flow end to end
@pytest.mark.parametrize("use_runner", [True, False], ids=["runner", "calls"])
def test_flat_frame_has_no_corners(monkeypatch, use_runner):
    """A flat frame has no FAST corners: Flow.predict returns ({}, None), as the reference does."""
    from fastmot_b200.flow import Flow
    from fastmot_b200.pool import TrackPool
    monkeypatch.setattr(Flow, "USE_RUNNER", use_runner)
    f = Flow((640, 480), scratch_floats=1 << 16)
    f.bind_pool(TrackPool(16))
    flat = np.full((480, 640, 3), 90, np.uint8)
    f.init(flat)
    assert f.predict(flat, []) == ({}, None)
    assert int(f.bg_count.item()) == 0


@pytest.mark.parametrize("use_runner", [True, False], ids=["runner", "calls"])
@pytest.mark.parametrize("size,scale,edge_row", [((1280, 720), (0.12, 0.12), 360), ((1920, 1080), (0.38, 0.38), 108)],
                         ids=["1280x720-0.12", "1920x1080-0.38"])
def test_flow_background_vs_oracle(monkeypatch, size, scale, edge_row, use_runner):
    """Flow.predict at background scales where the w / bw mask rule read the wrong frame row, with a track box whose
    top edge is that row: the background block of the point list equals the oracle's (cv2.resize + cv2 FAST) point for
    point, and H agrees at the end-to-end tier of tests/test_gpu_klt.py (LK is not bit-exact)."""
    from fastmot_b200 import MultiTracker
    from fastmot_b200.flow import Flow
    from fastmot_b200.synth import SyntheticScene
    from oracle.run import default_tracker_cfg
    from oracle.tracker import OracleTracker
    monkeypatch.setattr(Flow, "USE_RUNNER", use_runner)
    W, H = size
    cfg = default_tracker_cfg()
    cfg['flow_cfg'].bg_feat_scale_factor = scale
    scene = SyntheticScene(50, size=size, seed=14, label=0, dropout_frames=())
    tl, lb, cf, _ = scene.detections(0)
    edge_box = np.array([[W * 0.3, edge_row, W * 0.7, edge_row + 60.]])
    tl, lb, cf = np.concatenate([tl, edge_box]), np.append(lb, 0), np.append(cf, 0.9)
    # the mask row that reads frame row edge_row - 1 in cv2 read edge_row under the old rule
    bh = round(scale[1] * H)
    assert any(b == edge_row and a == edge_row - 1 for _, a, b in flipped(H, bh))
    trk = MultiTracker(size, 'cosine', **cfg)
    trk.reset(1 / 30)
    trk.init(scene.frame(0), _dets(tl, lb, cf))
    ora = OracleTracker(size, 'cosine', **cfg)
    ora.reset(1 / 30)
    ora.init(scene.frame(0), tl, lb)
    frame = scene.frame(1)
    ora.compute_flow(frame)
    dbg = ora.flow.debug
    active = [t for t in trk.tracks.values() if t.active]
    assert any(t.tlbr[1] == edge_row for t in active)
    dev = trk.pool.klt_ok.device
    h = torch.zeros(9, dtype=torch.float64, device=dev)
    ok = torch.zeros(1, dtype=torch.int32, device=dev)
    order = trk.flow.predict_device(torch.as_tensor(frame).cuda(), active, h, ok)
    torch.cuda.synchronize()
    assert (trk.flow._runner is not None) == use_runner
    meta = trk.flow.meta.cpu().numpy()
    want = dbg['all_prev'][dbg['bg_begin']:]
    assert meta[3] == 0 and meta[0] == dbg['bg_begin'] and meta[2] == len(want) > 50
    got = trk.flow.all_prev[meta[0]:meta[1]].cpu().numpy()
    np.testing.assert_array_equal(got, want)
    assert len(order) == len(active)
    assert int(ok.item()) == 1 and ora.homography is not None
    np.testing.assert_allclose(h.cpu().numpy().reshape(3, 3), ora.homography, atol=2e-3)
