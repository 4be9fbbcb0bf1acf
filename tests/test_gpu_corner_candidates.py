"""GPU: corner re-detection in boxes of any size.  A box with more than 4096 corner candidates (local maxima above the
quality threshold) runs the selection kernel's global-memory path; its kept corners must still be those of
cv2.goodFeaturesToTrack + the reference's filters (oracle/tracker.py, live on the host), with the tiers of
tests/test_gpu_klt.py and tests/test_gpu_flow_cfg.py.  The scenes and their candidate counts are pinned on the CPU in
tests/test_corner_candidates_cpu.py."""
from types import SimpleNamespace as NS

import numpy as np
import pytest
import torch

from oracle.flow_cfg_goldens import flow_cfg_namespace
from test_corner_candidates_cpu import (BOUNDARY_CROPS, BigObjectScene, boundary_scene, cfg_scene, large_box_scene,
                                        whole_frame_scene)

cv2 = pytest.importorskip("cv2")
pytestmark = pytest.mark.gpu


def _dets(tlbr, labels, conf):
    dt = np.dtype([('tlbr', float, 4), ('label', int), ('conf', float)], align=True)
    arr = np.zeros(len(tlbr), dt)
    arr['tlbr'], arr['label'], arr['conf'] = tlbr, labels, conf
    return arr.view(np.recarray)


def _cfg(flow_over=None, feat_over=None):
    from oracle.run import default_tracker_cfg
    cfg = default_tracker_cfg()
    cfg['flow_cfg'] = flow_cfg_namespace(cfg['flow_cfg'], flow_over or {}, feat_over or {})
    return cfg


def _keypoints(frame, tlbr, cfg):
    """One predict_device on `frame` after init on it: per track, nearest first, the GPU's kept corners and the
    oracle's, and the scratch floats the frame claimed."""
    from fastmot_b200 import MultiTracker
    from oracle.tracker import OracleTracker
    H, W = frame.shape[:2]
    labels, conf = np.zeros(len(tlbr), np.int64), np.full(len(tlbr), 0.9)
    trk = MultiTracker((W, H), 'cosine', **cfg)
    trk.reset(1 / 30)
    trk.init(frame, _dets(tlbr, labels, conf))
    active = [t for t in trk.tracks.values() if t.active]
    dev = trk.pool.klt_ok.device
    h = torch.zeros(9, dtype=torch.float64, device=dev)
    ok = torch.zeros(1, dtype=torch.int32, device=dev)
    order = trk.flow.predict_device(torch.as_tensor(frame).cuda(), active, h, ok)
    torch.cuda.synchronize()
    claimed = int(trk.flow.flags[0].item())
    begins = trk.flow.trk_begin[:len(order) + 1].cpu().numpy()
    pts = trk.flow.all_prev.cpu().numpy().reshape(-1, 2)
    got = [pts[begins[i]:begins[i + 1]] for i in range(len(order))]
    ora = OracleTracker((W, H), 'cosine', **cfg)
    ora.reset(1 / 30)
    ora.init(frame, tlbr, labels)
    ora_order = [t.trk_id for t in sorted(ora.tracks.values(), reverse=True)]
    ora.compute_flow(frame)          # drops every track when the camera motion fails (a box over the whole frame)
    dbg = ora.flow.debug
    assert ora_order == [tid for tid, _ in order]
    want = [dbg['all_prev'][dbg['begins'][i]:dbg['ends'][i]] for i in range(len(order))]
    return got, want, claimed


def _assert_exact(got, want):
    for i, (g, w) in enumerate(zip(got, want)):
        assert g.shape == w.shape and np.array_equal(g, w), (i, g.shape, w.shape)


def _crop_area(tlbr, W, H):
    x0, y0 = np.maximum(tlbr[:, 0], 0).astype(int), np.maximum(tlbr[:, 1], 0).astype(int)
    x1, y1 = np.minimum(tlbr[:, 2], W - 1).astype(int), np.minimum(tlbr[:, 3], H - 1).astype(int)
    return int(((x1 - x0 + 1) * (y1 - y0 + 1)).sum())


@pytest.mark.parametrize("feat_dist_factor", [0.06, 0.0])
def test_large_boxes_default_setting_vs_goodFeaturesToTrack(feat_dist_factor):
    """1000x1000 (about 43 000 candidates) and an occluded 640x640 box (about 6 000) at the default setting: every
    track keeps the oracle's corners, same set, same order."""
    frame, tlbr = large_box_scene()
    got, want, claimed = _keypoints(frame, tlbr, _cfg(dict(feat_dist_factor=feat_dist_factor)))
    _assert_exact(got, want)
    assert claimed > _crop_area(tlbr, 1920, 1080)        # the two large boxes took global candidate storage
    assert max(len(w) for w in want) > 100


@pytest.mark.parametrize("max_corners", [0, 1500])
@pytest.mark.parametrize("harris", [False, True])
@pytest.mark.parametrize("gs", [1, 5, 7])
@pytest.mark.parametrize("bs", [2, 5, 7])
def test_large_box_other_settings_vs_goodFeaturesToTrack(bs, gs, harris, max_corners):
    """Every other goodFeaturesToTrack setting on a box of more than 4096 candidates, minDistance 1 (maxCorners 0 keeps
    more than 1024 corners, fewer than the track's 4096 rows): the kept corners
    of tests/test_gpu_flow_cfg.py's tie tolerance, reused: per track at most one point in 500 (at least 1) differs,
    tied corners move at most 16 places, and every track but at most one is exact."""
    frame, tlbr = cfg_scene(bs, gs, harris)
    got, want, claimed = _keypoints(frame, tlbr, _cfg(dict(feat_dist_factor=0.0),
                                                      dict(blockSize=bs, gradientSize=gs, useHarrisDetector=harris,
                                                           k=0.04, maxCorners=max_corners)))
    assert claimed > 4 * _crop_area(tlbr, 1280, 720)
    exact = 0
    counts = []
    for i, (g, w) in enumerate(zip(got, want)):
        gs_, ws_ = set(map(tuple, g.tolist())), set(map(tuple, w.tolist()))
        assert len(gs_ ^ ws_) <= max(1, len(ws_) // 500), (i, g.shape, w.shape, len(gs_ ^ ws_))
        rank = {p: r for r, p in enumerate(q for q in map(tuple, w.tolist()) if q in gs_)}
        common = [q for q in map(tuple, g.tolist()) if q in ws_]
        shift = max((abs(r - rank[q]) for r, q in enumerate(common)), default=0)
        assert shift <= 16, (i, shift)
        exact += len(gs_ ^ ws_) == 0 and shift == 0
        counts.append(len(w))
    assert exact >= len(got) - 1, (exact, len(got))
    assert 1024 < max(counts) <= (4096 if max_corners == 0 else max_corners), counts


@pytest.mark.parametrize("n_cand", sorted(BOUNDARY_CROPS))
def test_boundary_candidate_counts_vs_goodFeaturesToTrack(n_cand):
    """Boxes of exactly 4095, 4096 and 4097 candidates keep the oracle's corners; up to 4096 the selection stays in
    shared memory (the frame claims only the response map's scratch), at 4097 it claims candidate storage."""
    frame, tlbr = boundary_scene(n_cand)
    got, want, claimed = _keypoints(frame, tlbr, _cfg())
    _assert_exact(got, want)
    w, h = BOUNDARY_CROPS[n_cand]
    if n_cand <= 4096:
        assert claimed == w * h, (claimed, w * h)
    else:
        assert claimed > w * h + 4 * n_cand, (claimed, w * h)


def test_whole_frame_box():
    """A 1920x1080 box of factor-3 texture (about 90 000 candidates): maxCorners 1000 keeps the oracle's corners; with
    maxCorners 0 and minDistance 1 it would keep more than its 4096 keypoint rows, and the tracker raises."""
    from fastmot_b200 import MultiTracker
    frame, tlbr = whole_frame_scene()
    trk = MultiTracker((1920, 1080), 'cosine', **_cfg())
    trk.reset(1 / 30)
    trk.init(frame, _dets(tlbr, np.zeros(1, np.int64), np.full(1, 0.9)))
    dev = trk.pool.klt_ok.device
    h = torch.zeros(9, dtype=torch.float64, device=dev)
    ok = torch.zeros(1, dtype=torch.int32, device=dev)
    trk.flow.predict_device(torch.as_tensor(frame).cuda(), [t for t in trk.tracks.values() if t.active], h, ok)
    torch.cuda.synchronize()
    got = trk.flow.all_prev[:int(trk.flow.trk_begin[1].item())].cpu().numpy()
    # no background is left for the camera motion, so OracleTracker stops before its keypoints: the reference's
    # goodFeaturesToTrack call on the whole frame (minDistance round(sqrt(area) * 0.06) = 86) + its ellipse filter
    gray = cv2.cvtColor(frame, cv2.COLOR_BGR2GRAY)
    kp = cv2.goodFeaturesToTrack(gray, 1000, 0.06, 86, blockSize=3).reshape(-1, 2)
    u = ((kp.astype(np.float64) - (959.5, 539.5)) / (960.0, 540.0)) ** 2
    want = kp[u.sum(1) <= 1.0]
    assert len(want) > 100
    np.testing.assert_array_equal(got, want)
    cfg = _cfg(dict(feat_dist_factor=0.0), dict(maxCorners=0))
    trk = MultiTracker((1920, 1080), 'cosine', **cfg)
    trk.reset(1 / 30)
    trk.init(frame, _dets(tlbr, np.zeros(1, np.int64), np.full(1, 0.9)))
    with pytest.raises(MemoryError, match="maxCorners") as e:
        trk.compute_flow(frame)
        trk.apply_kalman()
    assert "code 4" in str(e.value) and "code 3" not in str(e.value)


def test_scratch_too_small_raises():
    """scratch_floats that holds the response maps but not the large boxes' candidates: status 2, MemoryError."""
    from fastmot_b200 import MultiTracker
    frame, tlbr = large_box_scene()
    cfg = _cfg(dict(scratch_floats=_crop_area(tlbr, 1920, 1080) + 1000))
    trk = MultiTracker((1920, 1080), 'cosine', **cfg)
    trk.reset(1 / 30)
    trk.init(frame, _dets(tlbr, np.zeros(len(tlbr), np.int64), np.full(len(tlbr), 0.9)))
    with pytest.raises(MemoryError, match="code 2"):
        trk.compute_flow(frame)
        trk.apply_kalman()


def _run_tracker(scene, n_frames=12):
    """Per frame: homography, KLT boxes and keypoints after the flow step (frames >= 1), visible track boxes."""
    from fastmot_b200 import MultiTracker
    from oracle.run import default_tracker_cfg
    trk = MultiTracker(scene.size, 'cosine', **default_tracker_cfg())
    trk.reset(1 / 30)
    out = []
    for t in range(n_frames):
        frame = scene.frame(t)
        rec = {}
        if t == 0:
            tl, lb, cf, _ = scene.detections(0)
            trk.init(frame, _dets(tl, lb, cf))
        else:
            trk.compute_flow(frame)
            trk.apply_kalman()
            rec = dict(h=trk.homography.copy(), klt={k: v.copy() for k, v in trk.klt_bboxes.items()},
                       kps={k: v.keypoints.copy() for k, v in trk.tracks.items()})
            if t % 5 == 0:
                tl, lb, cf, ids = scene.detections(t)
                trk.update(t, _dets(tl, lb, cf), scene.embeddings(ids, t))
        rec['vis'] = {k: v.tlbr.copy() for k, v in trk.tracks.items() if v.confirmed and v.active}
        out.append(rec)
    return out


def test_end_to_end_big_object_vs_oracle():
    """12 frames at 1920x1080: 60 ordinary objects and a moving 1000x1000 one, detector every 5 frames: identical
    visible ID sets and boxes within +-1 px of OracleTracker."""
    from oracle.run import run_oracle_tracker
    scene = BigObjectScene()
    got = _run_tracker(scene)
    want, _ = run_oracle_tracker(scene, 12)
    for t in range(12):
        vis = got[t]['vis']
        w = dict(zip(want[t]['ids'].tolist(), want[t]['tlbr']))
        assert set(vis) == set(w), (t, set(vis) ^ set(w))
        for k in vis:
            assert np.abs(vis[k] - w[k]).max() <= 1.0, (t, k, vis[k], w[k])
    big_id, = [k for k, b in got[11]['vis'].items() if b[2] - b[0] > 900]
    assert len(got[10]['kps'][big_id]) > 100         # the large track keeps re-detected corners


def test_end_to_end_big_object_runner_equals_call_by_call(monkeypatch):
    """fm_flow_predict and the call-by-call sequence give bit-identical homographies, KLT boxes, keypoints and track
    boxes on the big-object sequence."""
    from fastmot_b200.flow import Flow
    scene = BigObjectScene()
    monkeypatch.setattr(Flow, "USE_RUNNER", True)
    a = _run_tracker(scene)
    monkeypatch.setattr(Flow, "USE_RUNNER", False)
    b = _run_tracker(scene)
    for t, (ra, rb) in enumerate(zip(a, b)):
        assert set(ra) == set(rb)
        if t:
            np.testing.assert_array_equal(ra['h'], rb['h'])
        for key in ('klt', 'kps', 'vis'):
            if key not in ra:
                continue
            assert set(ra[key]) == set(rb[key]), (t, key)
            for k in ra[key]:
                np.testing.assert_array_equal(ra[key][k], rb[key][k])


def test_mot_step_on_big_object():
    """MOT.step on frames with a 1000x1000 object of about 43 000 candidates (code 3 before the global path)."""
    from fastmot_b200 import MOT, DET_DTYPE
    from oracle.run import default_tracker_cfg
    scene = BigObjectScene()

    def dets(t):
        tl, lb, cf, _ = scene.detections(t)
        d = np.zeros(len(tl), DET_DTYPE)
        d['tlbr'], d['label'], d['conf'] = tl, lb, cf
        return d.view(np.recarray)

    mot = MOT(scene.size, detector_frame_skip=5, class_ids=(0,), yolo_detector_cfg=NS(model='YOLOv4Tiny'),
              feature_extractor_cfgs=(NS(model='OSNet025'),), tracker_cfg=NS(**default_tracker_cfg()),
              detections_override=dets, embeddings_override=lambda t, d: scene.embeddings(scene.detections(t)[3], t))
    mot.reset(1 / 30)
    for t in range(7):
        mot.step(scene.frame(t))
    assert mot.frame_count == 7
    assert len(list(mot.visible_tracks())) > 30
