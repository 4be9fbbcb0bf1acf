"""GPU: the KLT RANSAC kernels (csrc/klt_ransac.cu) against oracle/ransac.py, the NumPy restatement of OpenCV's RANSAC
that tests/test_oracle_ransac.py pins to cv2, at the batch, capacity, threshold and mask-chain edges.

Margin rule: random problems are checked to keep every point's float32 error under the oracle's model at least
1e-3 * thr^2 away from thr^2; masks, keypoints, counts and inlier ratios must then be bit-exact.  Boxes must be exact
wherever the unrounded coordinate is more than 1e-6 from a half-integer; H must map the frame corners within 1e-3 px
of the oracle's."""
from types import SimpleNamespace as NS

import numpy as np
import pytest
import torch

from oracle import ransac as R

pytestmark = pytest.mark.gpu

W, H = 1920, 1080
THR2 = 9.0
CORNERS = np.array([[0, 0, 1], [W - 1, 0, 1], [0, H - 1, 1], [W - 1, H - 1, 1.]])


def _lib():
    from fastmot_b200 import _lib
    return _lib, _lib.load()


def _margin_ok(err):
    return err is None or len(err) == 0 or bool((np.abs(err.astype(np.float64) - THR2) >= 1e-3 * THR2).all())


def _map(Hm, pts):
    q = pts @ np.asarray(Hm).T
    return q[:, :2] / q[:, 2:]


# ------------------------------------------------------------------------------------------------ homography
def run_homography(prev, cur, status, bg_begin, bg_end, max_iters=500, inlier_thresh=4, max_bg=None):
    from fastmot_b200.devmem import ptr, stream_ptr
    _l, lib = _lib()
    max_bg = max_bg or max(len(prev), 1)
    t = lambda a, dt: torch.as_tensor(np.ascontiguousarray(a, dt)).cuda()
    P, Cu, St = t(prev, np.float32), t(cur, np.float32), t(status, np.uint8)
    meta = t([bg_begin, bg_end, 0, 0], np.int32)
    good = torch.zeros(max_bg, dtype=torch.int32, device="cuda")
    inl = torch.zeros(max_bg, dtype=torch.int32, device="cuda")
    Hd = torch.zeros(9, dtype=torch.float64, device="cuda")
    ok = torch.full((1,), 7, dtype=torch.int32, device="cuda")
    kp = torch.zeros(max_bg, 2, dtype=torch.float32, device="cuda")
    kpp = torch.zeros(max_bg, 2, dtype=torch.float32, device="cuda")
    cnt = torch.full((1,), -1, dtype=torch.int32, device="cuda")
    _l.check(lib.fm_ransac_homography(ptr(P), ptr(Cu), ptr(St), ptr(meta), max_iters, 0.99, 3.0, inlier_thresh,
                                      ptr(good), ptr(inl), ptr(Hd), ptr(ok), ptr(kp), ptr(kpp), ptr(cnt), max_bg,
                                      stream_ptr()), "fm_ransac_homography")
    torch.cuda.synchronize()
    n = int(cnt.item())
    return NS(ok=int(ok.item()), H=Hd.cpu().numpy().reshape(3, 3), count=n, kp=kp[:max(n, 0)].cpu().numpy(),
              kp_prev=kpp[:max(n, 0)].cpu().numpy())


def _hom_points(rng, n, fo, noise=0.3):
    src = rng.uniform([0, 0], [W - 1, H - 1], (n, 2)).astype(np.float32)
    Ht = np.array([[1.003, 0.004, 3.5], [-0.002, 0.998, -2.25], [2e-6, -1e-6, 1.]])
    dst = _map(Ht, np.c_[src, np.ones(n)]) + rng.normal(0, noise, (n, 2))
    out = rng.random(n) < fo
    dst[out] += rng.uniform(15, 80, (int(out.sum()), 2)) * rng.choice([-1, 1], (int(out.sum()), 2))
    return src, dst.astype(np.float32)


def _hom_case(name):
    """(prev, cur, status, max_iters, inlier_thresh, max_bg) of a named case; the last point is the one the
    reference drops."""
    rng = np.random.default_rng(sum(map(ord, name)))
    st = None
    it, ithr, max_bg = 500, 4, None
    if name.startswith("count"):
        n = int(name[5:])
        src, dst = _hom_points(rng, n + 1, 0.0)
    elif name.startswith("inliers"):         # n_in exact inliers either side of the LM pair cache (1536)
        n_in = int(name[7:])
        src, dst = _hom_points(rng, n_in + 200, 0.0, noise=0.05)
        dst[n_in:] += np.float32(40)
        src, dst = np.concatenate([src, src[:1]]), np.concatenate([dst, dst[:1]])
    elif name == "max_bg":
        src, dst = _hom_points(rng, 2001, 0.1)
        max_bg = 2000
    elif name.startswith("iters"):
        it = int(name[5:])
        src, dst = _hom_points(rng, 400, 0.75)
    elif name == "lines":                    # three lines: checkSubset rejects every subset with 3 on one line
        x = rng.uniform(0, W - 1, 300)
        y = np.repeat([100., 500., 900.], 100)
        src = np.c_[x, y].astype(np.float32)
        dst = (src + [2.5, -1.5] + rng.normal(0, 0.3, src.shape)).astype(np.float32)
    elif name == "mirrored":                 # half the matches mirrored: the sign test rejects mixed quads
        src, dst = _hom_points(rng, 300, 0.0)
        dst[::2, 0] = np.float32(W - 1) - dst[::2, 0]
    elif name == "identical":                # getSubset exhausts its 10000 attempts on the first hypothesis
        src = np.full((50, 2), [300.5, 200.25], np.float32)
        dst = src + np.float32(2)
    elif name.startswith("thresh"):          # exactly 10 inliers of a translation, inlier_thresh 10 / 11
        ithr = int(name[6:])
        src = rng.uniform([0, 0], [W - 1, H - 1], (31, 2)).astype(np.float32)
        dst = src + np.float32(4)
        dst[10:] += rng.uniform(30, 90, (21, 2)).astype(np.float32)
    elif name == "status":                   # status-0 matches interleaved: good_idx keeps the order
        src, dst = _hom_points(rng, 700, 0.2)
        st = (rng.random(700) > 0.3).astype(np.uint8)
    else:
        raise KeyError(name)
    st = np.ones(len(src), np.uint8) if st is None else st
    return src, dst, st, it, ithr, max_bg


HOM_CASES = ["count3", "count4", "count5", "inliers1535", "inliers1536", "inliers1537", "max_bg", "iters1",
             "iters7", "iters8", "iters9", "iters500", "lines", "mirrored", "identical", "thresh10", "thresh11",
             "status"]


@pytest.mark.parametrize("name", HOM_CASES)
def test_homography_vs_oracle(name):
    src, dst, st, it, ithr, max_bg = _hom_case(name)
    lead = 17                                           # the background block starts after some track points
    prev = np.concatenate([np.zeros((lead, 2), np.float32), src])
    cur = np.concatenate([np.zeros((lead, 2), np.float32), dst])
    status = np.concatenate([np.zeros(lead, np.uint8), st])
    want = R.flow_homography(prev, cur, status, lead, len(prev), it, 0.99, 3.0, ithr)
    res = want["res"]
    if res is not None and res.ok:
        assert _margin_ok(res.err) and _margin_ok(R.homography_error(res.refined, prev[want["idx"]],
                                                                     cur[want["idx"]])), name
    got = run_homography(prev, cur, status, lead, len(prev), it, ithr, max_bg)
    assert got.ok == int(want["ok"]), name
    if not want["ok"]:
        assert got.count == 0
        return
    assert got.count == len(want["kp_idx"])
    np.testing.assert_array_equal(got.kp, cur[want["kp_idx"]])
    np.testing.assert_array_equal(got.kp_prev, prev[want["kp_idx"]])
    assert np.abs(_map(got.H, CORNERS) - _map(want["H"], CORNERS)).max() < 1e-3, name
    if name.startswith("iters") and int(name[5:]) < 500:
        assert res.iters == int(name[5:])                # the 75 % outlier count keeps niters above the cap


def test_homography_mask_is_the_refined_models():
    """The background keypoints are the matches within the threshold of the refined model (what findHomography
    returns), which here differ from the best hypothesis' inliers."""
    rng = np.random.default_rng(7)
    n = 600
    src = rng.uniform([0, 0], [W - 1, H - 1], (n, 2)).astype(np.float32)
    dst = (src * 1.01 + [4, -3] + rng.normal(0, 1.0, (n, 2))).astype(np.float32)
    dst[:60] += rng.uniform(20, 60, (60, 2)).astype(np.float32)
    prev, cur = np.concatenate([src, src[:1]]), np.concatenate([dst, dst[:1]])
    want = R.flow_homography(prev, cur, np.ones(n + 1, np.uint8), 0, n + 1)
    assert len(want["res"].final) != len(want["res"].inliers)
    got = run_homography(prev, cur, np.ones(n + 1, np.uint8), 0, n + 1)
    assert got.ok == 1 and got.count == len(want["kp_idx"])
    np.testing.assert_array_equal(got.kp, cur[want["kp_idx"]])


# ------------------------------------------------------------------------------------------------ affine partial
def run_affine(prev, cur, status, begins, slots, tlbr, max_iters=500, max_kp=1024, inlier_thresh=4, h_ok=None,
               cap=None):
    """One fm_ransac_affine_partial_batch call per 4 rounds until the fixed point, like Flow.finish_rounds.  tlbr:
    [n_trk][4] boxes in track order, stored at their slots."""
    from fastmot_b200.devmem import ptr, stream_ptr
    _l, lib = _lib()
    n = len(slots)
    cap = cap or (max(slots) + 1 if n else 1)
    t = lambda a, dt: torch.as_tensor(np.ascontiguousarray(a, dt)).cuda()
    P, Cu, St = t(prev, np.float32), t(cur, np.float32), t(status, np.uint8)
    tb, sl = t(begins, np.int32), t(slots if n else [0], np.int32)
    pool_tlbr = np.zeros((cap, 4))
    for k, s in enumerate(slots):
        pool_tlbr[s] = tlbr[k]
    tl = t(pool_tlbr, np.float64)
    flags = torch.zeros(16, dtype=torch.int32, device="cuda")
    est = torch.zeros(2 * max(n, 1) * 5, dtype=torch.int32, device="cuda")
    sig = torch.zeros(max(n, 1), dtype=torch.int64, device="cuda")
    klt = torch.full((cap, 4), -77., dtype=torch.float64, device="cuda")
    ok = torch.zeros(cap, dtype=torch.uint8, device="cuda")
    ratio = torch.full((cap,), -1., dtype=torch.float64, device="cuda")
    kp = torch.zeros(cap, max_kp, 2, dtype=torch.float32, device="cuda")
    kpp = torch.zeros(cap, max_kp, 2, dtype=torch.float32, device="cuda")
    cnt = torch.full((cap,), -1, dtype=torch.int32, device="cuda")
    hk = None if h_ok is None else t([h_ok], np.int32)
    rounds = 0
    while True:
        _l.check(lib.fm_ransac_affine_partial_batch(
            ptr(P), ptr(Cu), ptr(St), ptr(tb), ptr(sl), n, 4, ptr(flags), None if hk is None else ptr(hk), ptr(est),
            ptr(sig), ptr(tl), ptr(klt), ptr(ok), ptr(ratio), ptr(kp), ptr(kpp), ptr(cnt), max_kp, W, H, max_iters,
            0.99, 3.0, inlier_thresh, 10, rounds, stream_ptr()), "fm_ransac_affine_partial_batch")
        rounds += 4
        if int(flags[(rounds - 1) & 15].item()) == 0 or rounds >= 2 * max(n, 1) + 2:
            break
    torch.cuda.synchronize()
    return NS(ok=ok.cpu().numpy(), box=klt.cpu().numpy(), ratio=ratio.cpu().numpy(), kp=kp.cpu().numpy(),
              kp_prev=kpp.cpu().numpy(), count=cnt.cpu().numpy(), rounds=rounds)


def _check_affine(got, want, prev, cur, slots, max_kp, label="", margin=True):
    worst = 0.
    for k, (r, s) in enumerate(zip(want, slots)):
        if margin and r["res"] is not None and r["res"].ok:
            assert _margin_ok(r["res"].err), (label, k)
        assert got.ok[s] == int(r["ok"]), (label, k, r["m"])
        if not r["ok"]:
            assert got.count[s] in (0, -1), (label, k)
            continue
        n = min(len(r["kp_idx"]), max_kp)
        assert got.count[s] == n, (label, k)
        np.testing.assert_array_equal(got.kp[s, :n], cur[r["kp_idx"][:n]], err_msg=f"{label} {k}")
        np.testing.assert_array_equal(got.kp_prev[s, :n], prev[r["kp_idx"][:n]], err_msg=f"{label} {k}")
        assert got.ratio[s] == r["ratio"], (label, k)
        clear = np.abs(r["raw"] - np.floor(r["raw"]) - 0.5) > 1e-6
        np.testing.assert_array_equal(got.box[s][clear], r["box"][clear], err_msg=f"{label} {k}")
        worst = max(worst, float(np.abs(got.box[s] - r["box"]).max()))
    return worst


def _track(rng, box, n, fo=0.1, noise=0.3, scale=1.0, ang=0.0, shift=(2.5, -1.5)):
    p = rng.uniform(box[:2], box[2:] + 1, (n, 2)).astype(np.float32)
    Rm = scale * np.array([[np.cos(ang), -np.sin(ang)], [np.sin(ang), np.cos(ang)]])
    c = p @ Rm.T + shift + rng.normal(0, noise, (n, 2))
    out = rng.random(n) < fo
    c[out] += rng.uniform(10, 40, (int(out.sum()), 2)) * rng.choice([-1, 1], (int(out.sum()), 2))
    return p, c.astype(np.float32)


def _assemble(tracks):
    prev = np.concatenate([t[0] for t in tracks] + [np.zeros((1, 2), np.float32)])
    cur = np.concatenate([t[1] for t in tracks] + [np.zeros((1, 2), np.float32)])
    begins = np.cumsum([0] + [len(t[0]) for t in tracks])
    return prev, cur, begins


def _edge_tracks(rng):
    """Tracks in separate grid cells: filtered counts 2 / 3 / 4, 1023 / 1024 / 1025 points, identical points, scale
    at the clamp, a box leaving the frame, an empty segment."""
    specs = [dict(n=2), dict(n=3, fo=0), dict(n=4, fo=0), dict(n=1023), dict(n=1024), dict(n=1025),
             dict(n=40, same=True), dict(n=80, scale=0.89), dict(n=80, scale=0.91), dict(n=80, scale=1.09),
             dict(n=80, scale=1.11), dict(n=80, leave=True), dict(n=0), dict(n=200, fo=0.6), dict(n=200, fo=0.75)]
    tracks, boxes = [], []
    for i, sp in enumerate(specs):
        cx, cy = 120 + 230 * (i % 8), 200 + 500 * (i // 8)
        box = np.array([cx - 80., cy - 80, cx + 79, cy + 79])
        if sp.get("leave"):
            box = np.array([W - 60., 300, W + 99, 459])
        p, c = _track(rng, np.minimum(box, [W - 1, H - 1, W - 1, H - 1]), sp["n"], sp.get("fo", 0.1),
                      scale=sp.get("scale", 1.0), shift=(70., 0.) if sp.get("leave") else (2.5, -1.5))
        if sp.get("same"):
            p[:], c[:] = p[0], c[0]
        tracks.append((p, c))
        boxes.append(box)
    return tracks, boxes


@pytest.mark.parametrize("max_iters", [1, 31, 32, 33, 64, 500])
def test_affine_edges_vs_oracle(max_iters):
    rng = np.random.default_rng(100 + max_iters)
    tracks, boxes = _edge_tracks(rng)
    prev, cur, begins = _assemble(tracks)
    status = np.ones(len(prev), np.uint8)
    n = len(tracks)
    slots = list(rng.permutation(np.arange(3, 3 + 2 * n))[:n])      # slots permuted relative to track order
    want = R.flow_affine_serial(prev, cur, status, begins, boxes, (W, H), max_iters, max_pts=1024)
    got = run_affine(prev, cur, status, begins, slots, boxes, max_iters)
    _check_affine(got, want, prev, cur, slots, 1024, f"iters{max_iters}")
    assert want[5]["m"] == 1024 and want[5]["res"] is not None    # the 1025th point is past the capacity
    if max_iters < 500:
        assert want[14]["res"].iters == max_iters                     # 75 % outliers: the cap ends the loop
    assert not want[6]["ok"] and not want[11]["ok"] and not want[0]["ok"]


def test_affine_segment_beyond_capacity_keeps_first_points():
    """A segment longer than the kernel's per-track capacity (1024 points up to max_kp 1024, 4096 above) keeps its
    first filtered points.  Flow never builds one: a track carries at most max_kp keypoints."""
    rng = np.random.default_rng(5)
    tracks = [_track(rng, np.array([100., 100, 400, 400]), 1100, 0.3), _track(rng, np.array([700., 100, 1100, 500]),
                                                                              4096, 0.3)]
    prev, cur, begins = _assemble(tracks)
    status = np.ones(len(prev), np.uint8)
    boxes = [np.array([100., 100, 400, 400]), np.array([700., 100, 1100, 500])]
    want = R.flow_affine_serial(prev, cur, status, begins, boxes[:1], (W, H), max_pts=1024)
    got = run_affine(prev, cur, status, begins[:2], [0], boxes[:1], max_kp=1024)
    _check_affine(got, want, prev, cur, [0], 1024, "cap1024")
    want = R.flow_affine_serial(prev, cur, status, begins, boxes, (W, H), max_pts=4096)
    got = run_affine(prev, cur, status, begins, [0, 1], boxes, max_kp=4096)
    _check_affine(got, want, prev, cur, [0, 1], 4096, "cap4096")
    assert want[1]["m"] == 4096 and len(want[1]["kp_idx"]) > 1024


def test_affine_threshold_exact():
    """A dyadic translation of four square corners (every hypothesis from two inliers is exact), one match at squared
    error exactly 9 (inlier: the test is <=) and one at the next float above 9 (outlier)."""
    base = np.array([[96, 96], [104, 96], [96, 104], [104, 104]], np.float32) + np.float32(0.25)
    t = np.array([1.25, -0.5], np.float32)
    prev = np.concatenate([base, [[98.5, 99.75], [101.25, 97.5], [100.25, 100.75]]]).astype(np.float32)
    cur = prev + t
    cur[4] += [3, 0]                                      # err = 9
    cur[5] += [3, np.float32(2 ** -10)]                   # err = 9 + 2^-20 = nextafter(9, inf) in float
    cur[6] += [25, 31]
    e9 = R.affine_error(np.array([[1, 0, 1.25], [0, 1, -0.5]]), prev[4:6], cur[4:6])
    assert e9[0] == np.float32(9) and e9[1] == np.nextafter(np.float32(9), np.float32(10))
    res = R.run(prev, cur, "affine", record=True)
    for idx, model in res.hypotheses:
        if max(idx) < 4:
            np.testing.assert_array_equal(model, [[1, 0, 1.25], [0, 1, -0.5]])
    np.testing.assert_array_equal(res.model, [[1, 0, 1.25], [0, 1, -0.5]])
    np.testing.assert_array_equal(res.inliers, [0, 1, 2, 3, 4])
    box = [np.array([90., 90, 110, 110])]
    want = R.flow_affine_serial(prev, cur, np.ones(7, np.uint8), [0, 7], box, (W, H))
    got = run_affine(prev, cur, np.ones(7, np.uint8), [0, 7], [0], box)
    _check_affine(got, want, prev, cur, [0], 1024, "thr", margin=False)
    assert got.count[0] == 5


def test_affine_error_in_float_like_opencv():
    """Matches whose squared error lies within one float rounding of 9, where the double residual and OpenCV's float
    one disagree (tests/test_oracle_ransac.py pins cv2 to the float one): the kernel's mask is the float one."""
    rng = np.random.default_rng(3)
    n_in, n_probe = 40, 12
    src = rng.uniform(100, 900, (n_in + n_probe, 2)).astype(np.float32)
    c, s = 0.98 * np.cos(0.03), 0.98 * np.sin(0.03)
    dst = (src @ np.array([[c, s], [-s, c]]) + [7.3, -4.1] + rng.normal(0, 0.3, src.shape)).astype(np.float32)
    dst[n_in:] += 3.0
    best = R.run(src, dst, "affine").model
    for i in range(n_in, n_in + n_probe):
        th = rng.uniform(0, 2 * np.pi)
        b0 = best[:, :2] @ src[i].astype(np.float64) + best[:, 2]
        for k in range(-4000, 4000):
            cand = (b0 + (3.0 + k * 2e-7) * np.array([np.cos(th), np.sin(th)])).astype(np.float32)[None]
            if (R.affine_error(best, src[i:i + 1], cand, "float")[0] <= 9) != (
                    R.affine_error(best, src[i:i + 1], cand, "double")[0] <= 9):
                dst[i] = cand[0]
                break
    fl = R.run(src, dst, "affine")
    db = R.run(src, dst, "affine", affine_precision="double")
    assert not np.array_equal(fl.mask, db.mask)
    prev, cur = np.concatenate([src, src[:1]]), np.concatenate([dst, dst[:1]])
    n = len(src)
    box = [np.array([100., 100, 900, 900])]
    got = run_affine(prev, cur, np.ones(n + 1, np.uint8), [0, n], [0], box)
    assert got.ok[0] == 1
    m = int(got.count[0])
    np.testing.assert_array_equal(got.kp[0, :m], dst[fl.inliers])


def test_affine_h_ok_zero_writes_nothing():
    rng = np.random.default_rng(9)
    tracks = [_track(rng, np.array([100., 100, 300, 300]), 100)]
    prev, cur, begins = _assemble(tracks)
    got = run_affine(prev, cur, np.ones(len(prev), np.uint8), begins, [2], [np.array([100., 100, 300, 300])],
                     h_ok=0)
    assert got.ok.sum() == 0 and (got.box == -77.).all() and (got.count == -1).all()


# ------------------------------------------------------------------------------------------------ mask chains
def _chains(rng, lengths):
    """Chains of tracks along rows: each track's predicted box covers the left part of the next track's points."""
    tracks, boxes = [], []
    for row, L in enumerate(lengths):
        y0 = 40 + 200 * row
        for k in range(L):
            x0 = 20 + 40 * k
            box = np.array([x0, y0, x0 + 69., y0 + 69])
            tracks.append(_track(rng, box, 60, 0.1, shift=(3.0, 1.0)))
            boxes.append(box)
    return tracks, boxes


def _flow_rounds(tracks, boxes, slots):
    """Runs the affine rounds through Flow as predict_device does: ROUNDS_AHEAD rounds, then finish_rounds."""
    from fastmot_b200.flow import Flow
    from fastmot_b200.pool import TrackPool
    from oracle.run import default_tracker_cfg
    f = Flow((W, H), **vars(default_tracker_cfg()['flow_cfg']))
    f.bind_pool(TrackPool(256))
    prev, cur, begins = _assemble(tracks)
    P, n = len(prev), len(tracks)
    f.all_prev[:P].copy_(torch.as_tensor(prev))
    f.all_cur[:P].copy_(torch.as_tensor(cur))
    f.status[:P] = 1
    f.trk_begin[:n + 1].copy_(torch.as_tensor(begins.astype(np.int32)))
    f.slots_dev[:n].copy_(torch.as_tensor(np.int32(slots)))
    for k, s in enumerate(slots):
        f.pool.tlbr[s] = torch.as_tensor(boxes[k])
    f.pool.klt_ok.zero_()
    f.flags.zero_()
    f._affine_args = (n, W, H)
    rounds = 0
    for _ in range(Flow.ROUNDS_AHEAD // 4):
        rounds = f._enqueue_rounds(rounds, 4)
    rounds = f.finish_rounds(rounds)
    torch.cuda.synchronize()
    pool = f.pool
    got = NS(ok=pool.klt_ok.cpu().numpy(), box=pool.klt_tlbr.cpu().numpy(), ratio=pool.inlier_ratio.cpu().numpy(),
             kp=pool.kp.cpu().numpy(), kp_prev=pool.kp_prev.cpu().numpy(), count=pool.kp_count.cpu().numpy(),
             rounds=rounds)
    return got, prev, cur, begins


@pytest.mark.parametrize("lengths", [(1,), (8,), (9,), (1, 8, 9, 40)])
def test_mask_chains_through_flow_rounds(lengths):
    rng = np.random.default_rng(sum(lengths))
    tracks, boxes = _chains(rng, lengths)
    slots = list(np.random.default_rng(1).permutation(256)[:len(tracks)])
    got, prev, cur, begins = _flow_rounds(tracks, boxes, slots)
    want = R.flow_affine_serial(prev, cur, np.ones(len(prev), np.uint8), begins, boxes, (W, H))
    _check_affine(got, want, prev, cur, slots, 1024, f"chain{lengths}")
    masked = sum(r["m"] < 60 for r in want)
    assert masked >= sum(lengths) - len(lengths) - 2           # every track but a chain's first loses points


def test_bulk_random_tracks_vs_oracle():
    """About 300 tracks of random size, motion, outlier fraction and overlap in one launch."""
    rng = np.random.default_rng(2024)
    tracks, boxes = [], []
    while len(tracks) < 300:
        w, h = rng.uniform(20, 200, 2)
        x0, y0 = rng.uniform([-30, -30], [W - 20, H - 20])
        box = np.rint([x0, y0, x0 + w, y0 + h])
        n = int(rng.choice([0, 2, 3, 5, 12, 40, 150, 600]))
        t = _track(rng, np.clip(box, 0, [W - 1, H - 1, W - 1, H - 1]), n, rng.choice([0, .1, .5, .7]),
                   noise=rng.uniform(0.05, 0.8), scale=rng.uniform(0.85, 1.15), ang=rng.uniform(-0.1, 0.1),
                   shift=rng.uniform(-10, 10, 2))
        tracks.append(t)
        boxes.append(box)
    prev, cur, begins = _assemble(tracks)
    status = (rng.random(len(prev)) > 0.05).astype(np.uint8)
    slots = list(rng.permutation(400)[:300])
    want = R.flow_affine_serial(prev, cur, status, begins, boxes, (W, H))
    got = run_affine(prev, cur, status, begins, slots, boxes)
    worst = _check_affine(got, want, prev, cur, slots, 1024, "bulk")
    print(f"bulk: {sum(r['ok'] for r in want)} of 300 tracks predicted, worst box deviation {worst} px, "
          f"{got.rounds} rounds")
