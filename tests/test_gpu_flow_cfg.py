"""GPU parity of the KLT stage at other frame sizes, optical-flow scales and goodFeaturesToTrack settings, with the tiers
of tests/test_gpu_klt.py: integer image ops bit-exact against OpenCV 4.13; the kept corners those of
cv2.goodFeaturesToTrack + the reference's filters, in the same order up to float-precision ties; end to end identical
visible ID sets and boxes within +-1 px against tests/golden/seq_flow_cfg.npz (the unmodified reference,
oracle/flow_cfg_goldens.py)."""
import os
from types import SimpleNamespace as NS

import numpy as np
import pytest
import torch

from conftest import GOLDEN
from test_flow_cfg_oracle import RESIZE_SCALES, RESIZE_SIZES, flow_case_cfg
from oracle.flow_cfg_goldens import FLOW_CFG_CASES, flow_cfg_namespace

cv2 = pytest.importorskip("cv2")
pytestmark = pytest.mark.gpu


def _dets(tlbr, labels, conf):
    dt = np.dtype([('tlbr', float, 4), ('label', int), ('conf', float)], align=True)
    arr = np.zeros(len(tlbr), dt)
    arr['tlbr'], arr['label'], arr['conf'] = tlbr, labels, conf
    return arr.view(np.recarray)


@pytest.mark.parametrize("size", RESIZE_SIZES, ids=[f"{w}x{h}" for w, h in RESIZE_SIZES])
def test_gray_resize_pyramid_scharr_exact(size):
    """Gray, optical-flow image, pyramid levels and Scharr images of Flow._preprocess against cv2.cvtColor +
    cv2.resize + cv2.buildOpticalFlowPyramid, at every scale of the CPU restatement test."""
    from fastmot_b200.flow import Flow
    from fastmot_b200.synth import SyntheticScene
    frame = SyntheticScene(60, size=size, seed=6).frame(2)
    gray = cv2.cvtColor(frame, cv2.COLOR_BGR2GRAY)
    frame_dev = torch.as_tensor(frame).cuda()
    for scale in RESIZE_SCALES:
        f = Flow(size, opt_flow_scale_factor=scale, scratch_floats=1 << 10)
        f._preprocess(frame_dev, 0)
        torch.cuda.synchronize()
        assert np.array_equal(f.gray[0].cpu().numpy(), gray)
        sw, sh = f.opt_flow_sz
        assert (sw, sh) == (round(scale[0] * size[0]), round(scale[1] * size[1]))
        small = cv2.resize(gray, (sw, sh))
        assert np.array_equal(f.pyr[0][0].cpu().numpy(), small), (size, scale)
        n, pyr = cv2.buildOpticalFlowPyramid(small, (5, 5), 5, withDerivatives=True)
        assert n + 1 == len(f.level_sizes), (size, scale)
        for lvl in range(n + 1):
            assert np.array_equal(f.pyr[0][lvl].cpu().numpy(), pyr[2 * lvl]), (size, scale, lvl)
            assert np.array_equal(f.deriv[0][lvl].cpu().numpy(), pyr[2 * lvl + 1]), (size, scale, lvl)
        del f


# ------------------------------------------------------------------------------------------------ keypoints
def _corner_scene(bs, gs, harris):
    """A 1280x720 frame with one large fine-textured box (sized so that about 2800 local maxima pass the quality
    threshold under this goodFeaturesToTrack setting: more than 1024 corners kept, fewer than the 4096-candidate cap)
    and ten ordinary boxes, two of them occluding the large one."""
    from fastmot_b200.synth import smooth_texture
    rng = np.random.default_rng(17)
    W, H = 1280, 720
    frame = smooth_texture(rng, H, W, 10)
    fine = smooth_texture(rng, 420, 420, 3)
    g = cv2.cvtColor(fine, cv2.COLOR_BGR2GRAY)
    eig = cv2.cornerHarris(g, bs, gs, 0.04) if harris else cv2.cornerMinEigenVal(g, bs, ksize=gs)
    e = np.where(eig > eig.max() * 0.06, eig, 0)
    density = ((e != 0) & (e == cv2.dilate(e, None))).mean()
    side = int(min(420, np.sqrt(2800 / density)))
    boxes = [(30, 30, side, side)]
    frame[30:30 + side, 30:30 + side] = fine[:side, :side]
    for i in range(10):
        x, y = 480 + 75 * (i % 5), 60 + 220 * (i // 5)
        if i >= 8:
            x, y = 30 + side - 40 - 60 * (i - 8), 30 + side - 50
        w, h = 56, 96
        frame[y:y + h, x:x + w] = smooth_texture(rng, h, w, 6)
        boxes.append((x, y, w, h))
    tlbr = np.array([(x, y, x + w - 1, y + h - 1) for x, y, w, h in boxes], np.float64)
    return frame, tlbr


@pytest.mark.parametrize("max_corners", [0, 1500])
@pytest.mark.parametrize("harris", [False, True])
@pytest.mark.parametrize("gs", [1, 5, 7])
@pytest.mark.parametrize("bs", [2, 5, 7])
def test_keypoint_maintenance_vs_goodFeaturesToTrack_cfg(bs, gs, harris, max_corners):
    """For every track -- nearest first, each one masking the next -- the corners the GPU keeps are the points
    cv2.goodFeaturesToTrack(blockSize, gradientSize, useHarrisDetector, maxCorners, minDistance 1) + the reference's
    filters keep, in the same order, for every track but at most one, which may differ by float-precision ties; one
    track keeps more than 1024."""
    from fastmot_b200 import MultiTracker
    from oracle.run import default_tracker_cfg
    from oracle.tracker import OracleTracker
    cfg = default_tracker_cfg()
    cfg['flow_cfg'] = flow_cfg_namespace(cfg['flow_cfg'], dict(feat_dist_factor=0.0),
                                         dict(blockSize=bs, gradientSize=gs, useHarrisDetector=harris, k=0.04,
                                              maxCorners=max_corners))
    frame, tlbr = _corner_scene(bs, gs, harris)
    labels, conf = np.zeros(len(tlbr), np.int64), np.full(len(tlbr), 0.9)
    trk = MultiTracker((1280, 720), 'cosine', **cfg)
    trk.reset(1 / 30)
    trk.init(frame, _dets(tlbr, labels, conf))
    ora = OracleTracker((1280, 720), 'cosine', **cfg)
    ora.reset(1 / 30)
    ora.init(frame, tlbr, labels)
    ora.compute_flow(frame)
    dbg = ora.flow.debug
    active = [t for t in trk.tracks.values() if t.active]
    dev = trk.pool.klt_ok.device
    h = torch.zeros(9, dtype=torch.float64, device=dev)
    ok = torch.zeros(1, dtype=torch.int32, device=dev)
    order = trk.flow.predict_device(torch.as_tensor(frame).cuda(), active, h, ok)
    torch.cuda.synchronize()
    begins = trk.flow.trk_begin[:len(order) + 1].cpu().numpy()
    pts = trk.flow.all_prev.cpu().numpy().reshape(-1, 2)
    assert [t.trk_id for t in sorted(ora.tracks.values(), reverse=True)] == [tid for tid, _ in order]
    counts = []
    exact = 0
    for i, (tid, _) in enumerate(order):
        got = pts[begins[i]:begins[i + 1]]
        want = dbg['all_prev'][dbg['begins'][i]:dbg['ends'][i]]
        # the response's float sums run in another order than OpenCV's filters: a corner whose response ties a
        # neighbour's or the quality threshold to float precision may be decided the other way (seen: one corner of
        # 1240 at blockSize 2, aperture 7), and tied corners may swap places -- only locally
        gs_, ws_ = set(map(tuple, got.tolist())), set(map(tuple, want.tolist()))
        assert len(gs_ ^ ws_) <= max(1, len(ws_) // 500), (tid, got.shape, want.shape, len(gs_ ^ ws_))
        rank = {p: r for r, p in enumerate(q for q in map(tuple, want.tolist()) if q in gs_)}
        common = [q for q in map(tuple, got.tolist()) if q in ws_]
        shift = max((abs(r - rank[q]) for r, q in enumerate(common)), default=0)
        assert shift <= 16, (tid, shift)
        exact += len(gs_ ^ ws_) == 0 and shift == 0
        counts.append(len(want))
    assert exact >= len(order) - 1, (exact, len(order))
    if max_corners == 0:
        assert max(counts) > 1024, counts
    else:
        assert max(counts) <= max_corners
    bg_got = pts[begins[len(order)]:begins[len(order)] + (len(dbg['all_prev']) - dbg['bg_begin'])]
    assert np.array_equal(bg_got, dbg['all_prev'][dbg['bg_begin']:])


# ------------------------------------------------------------------------------------------------ end to end
@pytest.mark.parametrize("i", range(len(FLOW_CFG_CASES)), ids=[c[0] for c in FLOW_CFG_CASES])
def test_end_to_end_tracker_with_klt_vs_reference_flow_cfg_golden(i):
    """Full MultiTracker (KLT on GPU) on each golden case: identical visible ID sets, boxes within +-1 px, KLT box id
    sets and H as in test_gpu_klt.py's default-configuration test."""
    from fastmot_b200 import MultiTracker
    from fastmot_b200.synth import SyntheticScene
    g = np.load(os.path.join(GOLDEN, "seq_flow_cfg.npz"))
    _, scene_kw, n_frames, _, _ = FLOW_CFG_CASES[i]
    scene = SyntheticScene(**scene_kw)
    trk = MultiTracker(scene.size, 'cosine', **flow_case_cfg(i))
    trk.reset(1 / 30)
    exact = total = 0
    for t in range(n_frames):
        frame = scene.frame(t)
        if t == 0:
            tlbr, labels, conf, ids = scene.detections(0)
            trk.init(frame, _dets(tlbr, labels, conf))
        else:
            trk.compute_flow(frame)
            trk.apply_kalman()
            assert trk.homography is not None, t
            np.testing.assert_allclose(trk.homography, g[f'c{i}_H_{t}'], atol=2e-3), t
            want_ids = set(int(k) for k in g[f'c{i}_klt_ids_{t}'])
            assert len(set(trk.klt_bboxes) ^ want_ids) <= max(1, len(want_ids) // 50), t
            if t % 5 == 0:
                tlbr, labels, conf, ids = scene.detections(t)
                trk.update(t, _dets(tlbr, labels, conf), scene.embeddings(ids, t))
        vis = {k: v.tlbr for k, v in trk.tracks.items() if v.confirmed and v.active}
        want = dict(zip(g[f'c{i}_vis_ids_{t}'].tolist(), g[f'c{i}_vis_tlbr_{t}']))
        assert set(vis) == set(want), (t, set(vis) ^ set(want))
        for k in vis:
            d = np.abs(vis[k] - want[k]).max()
            assert d <= 1.0, (t, k, vis[k], want[k])
            exact += d == 0
            total += 1
    assert exact / max(total, 1) > 0.7, exact / max(total, 1)


@pytest.mark.parametrize("i", range(len(FLOW_CFG_CASES)), ids=[c[0] for c in FLOW_CFG_CASES])
def test_flow_runner_equals_call_by_call_sequence_cfg(i, monkeypatch):
    """fm_flow_predict (gray_resize / keypoints_cfg chosen inside the runner) enqueues what the call-by-call sequence
    of Flow.predict_device enqueues at each golden case's size and flow_cfg: identical homographies, KLT boxes,
    keypoints and track boxes, bit for bit."""
    from fastmot_b200 import MultiTracker
    from fastmot_b200.flow import Flow
    from fastmot_b200.synth import SyntheticScene
    _, scene_kw, _, _, _ = FLOW_CFG_CASES[i]
    scene = SyntheticScene(**scene_kw)
    frames = [scene.frame(t) for t in range(12)]

    def run(use_runner):
        monkeypatch.setattr(Flow, "USE_RUNNER", use_runner)
        trk = MultiTracker(scene.size, 'cosine', **flow_case_cfg(i))
        trk.reset(1 / 30)
        out = []
        for t, frame in enumerate(frames):
            if t == 0:
                tl, lb, cf, _ = scene.detections(0)
                trk.init(frame, _dets(tl, lb, cf))
                continue
            trk.compute_flow(frame)
            assert (trk.flow._runner is not None) == use_runner
            trk.apply_kalman()
            klt = trk.klt_bboxes
            kps = {k: v.keypoints.copy() for k, v in trk.tracks.items()}
            if t % 5 == 0:
                tl, lb, cf, ids = scene.detections(t)
                trk.update(t, _dets(tl, lb, cf), scene.embeddings(ids, t))
            out.append((trk.homography.copy(), {k: v.copy() for k, v in klt.items()}, kps,
                        {k: v.tlbr.copy() for k, v in trk.tracks.items()}))
        return out

    a, b = run(True), run(False)
    assert len(a) == len(b) == 11
    for (ha, ka, pa, ta), (hb, kb, pb, tb) in zip(a, b):
        np.testing.assert_array_equal(ha, hb)
        assert set(ka) == set(kb) and len(ka) > 30
        for k in ka:
            np.testing.assert_array_equal(ka[k], kb[k])
        assert set(pa) == set(pb)
        for k in pa:
            np.testing.assert_array_equal(pa[k], pb[k])
        assert set(ta) == set(tb)
        for k in ta:
            np.testing.assert_array_equal(ta[k], tb[k])


def test_multicamera_odd_size_camera_equals_separate_mot(monkeypatch):
    """A 1920x1080 + 1173x880 MultiCameraMOT group with the default flow_cfg: each camera's visible tracks (ids and
    boxes, bit for bit) are those of a separate MOT of its size."""
    from fastmot_b200 import MOT, MultiCameraMOT
    from fastmot_b200.synth import SyntheticScene
    from oracle.run import default_tracker_cfg
    from test_gpu_multistream import _dets_fn
    from test_gpu_yolo_ops import CASES
    bias, gain, _ = CASES['YOLOv4Tiny']
    monkeypatch.setenv("FM_SYNTH_OBJ_BIAS", str(bias))
    monkeypatch.setenv("FM_SYNTH_HEAD_GAIN", str(gain))
    sizes = [(1920, 1080), (1173, 880)]
    scenes = [SyntheticScene(64, size=wh, seed=3 + 101 * s) for s, wh in enumerate(sizes)]
    dets = [_dets_fn(sc) for sc in scenes]
    T = 13
    frames = [[sc.frame(t) for sc in scenes] for t in range(T)]
    kw = dict(detector_frame_skip=5, class_ids=(0,), yolo_detector_cfg=NS(model='YOLOv4Tiny'),
              feature_extractor_cfgs=(NS(model='OSNet025'),), tracker_cfg=NS(**default_tracker_cfg()))

    def emb(s, t):
        return scenes[s].embeddings(scenes[s].detections(t)[3], t)

    want = [[None] * T for _ in sizes]
    for s, wh in enumerate(sizes):
        mot = MOT(wh, detections_override=lambda i, s=s: dets[s](i),
                  embeddings_override=lambda i, d, s=s: emb(s, i), **kw)
        mot.reset(1 / 30)
        for t in range(T):
            mot.step(frames[t][s])
            want[s][t] = {trk.trk_id: trk.tlbr.copy() for trk in mot.visible_tracks()}
        del mot
    mc = MultiCameraMOT(sizes, detections_override=lambda s, i: dets[s](i),
                        embeddings_override=lambda s, i, d: emb(s, i), **kw)
    mc.reset(1 / 30)
    for t in range(T):
        mc.step(frames[t])
        for s in range(len(sizes)):
            vis = {trk.trk_id: trk.tlbr for trk in mc.visible_tracks(s)}
            assert set(vis) == set(want[s][t]), (s, t, set(vis) ^ set(want[s][t]))
            for k in vis:
                assert np.array_equal(vis[k], want[s][t][k]), (s, t, k)
    assert len(want[1][T - 1]) >= 20
