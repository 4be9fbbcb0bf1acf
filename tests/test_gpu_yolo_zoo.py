"""GPU checks of the seven YOLO models added to the first four (YOLOv3, YOLOv3-SPP, YOLOv3-tiny, YOLOv4x-mish,
YOLOv4-csp-swish, YOLOv4-csp-x-swish, YOLOv4-P6) at the reference's input sizes: every engine launch against the
float64 reference (test_gpu_yolo_ops.run_launch_by_launch), the head decode and NMS on the engines' own heads, graph
replay, Darknet files, the detector end to end, and the heads coarsest first (v3) and four heads (P6) through the
one-image, batched and per-image-geometry detect paths."""
import os
import time
from types import SimpleNamespace as NS

import numpy as np
import pytest
import torch

import test_gpu_yolo_ops as ops
from conftest import GOLDEN

pytestmark = pytest.mark.gpu

# model -> synthetic head objectness bias and head gain (on the scene frame about 680 / 1170 / 710 / 540 / 1080 / 1170 /
# 1080 candidates pass conf_thresh), the (kind, conv path) pairs its launches reach
_SCALED = {('conv', 'tc'), ('conv', 'tma'), ('conv+shortcut', 'tc'), ('conv+shortcut', 'tma'), ('maxpool', None),
           ('upsample', None)}
ZOO = {
    'YOLOv3': (-2.0, 1.0, {('conv', 'tc'), ('conv', 'tma'), ('conv+shortcut', 'tc'), ('conv+shortcut', 'tma'),
                           ('copy', None), ('upsample', None)}),
    'YOLOv3SPP': (-3.0, 1.0, {('conv', 'tc'), ('conv', 'tma'), ('conv+shortcut', 'tc'), ('conv+shortcut', 'tma'),
                              ('copy', None), ('maxpool', None), ('upsample', None)}),
    'YOLOv3Tiny': (-1.0, 1.0, {('conv', 'tc'), ('conv', 'tma'), ('maxpool', None), ('upsample', None)}),
    'YOLOv4xMish': (-8.0, 0.05, _SCALED),
    'YOLOv4CSPSwish': (-5.0, 0.25, _SCALED),
    'YOLOv4CSPxSwish': (-20.0, 0.015, _SCALED),
    'YOLOv4P6': (-8.0, 0.015, _SCALED),
}


def _weights(name):
    from fastmot_b200 import models
    from fastmot_b200.models import darknet
    bias, gain, _ = ZOO[name]
    m = models.YOLO.get_model(name)
    layers = darknet.BUILDERS[m.CFG](num_classes=m.NUM_CLASSES, anchors_per_head=len(m.ANCHORS[0]) // 2)
    return m, layers, darknet.synthetic_weights(layers, 3, head_obj_bias=bias, num_classes=m.NUM_CLASSES,
                                                head_gain=gain)


def _synth_env(monkeypatch, name):
    """build_yolo_engine's synthetic heads at this file's bias / gain (inside key_cap on the synthetic scenes)."""
    bias, gain, _ = ZOO[name] if name in ZOO else ops.CASES[name]
    monkeypatch.setenv("FM_SYNTH_OBJ_BIAS", str(bias))
    monkeypatch.setenv("FM_SYNTH_HEAD_GAIN", str(gain))


class ZooCase:
    """test_gpu_yolo_ops.Case for this file's models: the eager engine, its detector and the scene frame's heads."""

    def __init__(self, name):
        from fastmot_b200.detector import YOLODetector
        from fastmot_b200.engine import YoloEngine
        from fastmot_b200.synth import SyntheticScene
        self.name, self.expect = name, ZOO[name][2]
        m, self.layers, self.weights = _weights(name)
        self.model = m
        self.eng = YoloEngine(self.layers, m.INPUT_SHAPE[1:], self.weights, use_graph=False)
        self.det = YOLODetector((1920, 1080), tuple(range(m.NUM_CLASSES)), name, engine=self.eng)
        self.det.preprocess(torch.as_tensor(SyntheticScene(200, seed=3).frame(0)).cuda())
        self.eng.forward(self.det.inp)
        torch.cuda.synchronize()

    def close(self):
        self.eng = self.det = None
        torch.cuda.empty_cache()


@pytest.fixture(scope="module", params=list(ZOO))
def zcase(request):
    c = ZooCase(request.param)
    yield c
    c.close()


# ------------------------------------------------------------------------------------------------ engine
def test_zoo_engine_launch_by_launch(zcase):
    """Input bit-checks, out-of-view checks and float64 values of every launch (P6 at 1280 included)."""
    t0 = time.time()
    eng = zcase.eng
    reached = {(e.kind, e.info.get('path')) for e in eng.trace}
    assert reached == zcase.expect, reached
    assert eng.n_simt == 0
    ops._report(zcase.name, eng, ops.run_launch_by_launch(eng, zcase.name), t0)


def test_zoo_decode_of_engine_heads(zcase):
    ops.test_decode_of_engine_heads(zcase)


def test_zoo_nms_of_engine_candidates_teacher_forced(zcase):
    ops.test_nms_of_engine_candidates_teacher_forced(zcase)


@pytest.mark.parametrize("name", ['YOLOv3', 'YOLOv4P6'])
def test_graph_replay_matches_eager(name):
    from fastmot_b200.engine import YoloEngine
    m, layers, weights = _weights(name)
    hw = m.INPUT_SHAPE[1:]
    a = YoloEngine(layers, hw, weights, use_graph=False)
    b = YoloEngine(layers, hw, weights, use_graph=True)
    x = torch.rand(*hw, 8, device="cuda").half()
    x[..., 3:] = 0
    ha = [h.clone() for h in a.forward(x)]
    for _ in range(3):
        hb = b.forward(x)
    torch.cuda.synchronize()
    assert len(ha) == len(hb) == len(m.LAYER_FACTORS)
    for p, q in zip(ha, hb):
        assert torch.equal(p.view(torch.int16), q.view(torch.int16))


@pytest.mark.parametrize("name", ['YOLOv3Tiny', 'YOLOv4P6'])
def test_darknet_files_give_the_builder_heads_bit_for_bit(name, tmp_path):
    """.cfg + .weights written to disk and loaded back: the identity batch norm save_weights writes folds to a scale of
    exactly 1, so the device weights and the heads equal the builder path's bit for bit."""
    from fastmot_b200.engine import YoloEngine
    from fastmot_b200.models import darknet
    m, layers, weights = _weights(name)
    _, H, W = m.INPUT_SHAPE
    (tmp_path / "net.cfg").write_text(darknet.to_cfg(layers, W, H))
    darknet.save_weights(str(tmp_path / "net.weights"), layers, weights, 3)
    net, layers2 = darknet.parse_cfg((tmp_path / "net.cfg").read_text())
    loaded = darknet.load_weights(str(tmp_path / "net.weights"), layers2, 3)
    a = YoloEngine(layers, (net['height'], net['width']), weights, use_graph=False)
    b = YoloEngine(layers2, (net['height'], net['width']), loaded, use_graph=False)
    for i in a.params:
        assert torch.equal(a.params[i][0].view(torch.int16), b.params[i][0].view(torch.int16)), i
        assert torch.equal(a.params[i][1], b.params[i][1]), i
    x = torch.rand(H, W, 8, device="cuda").half()
    x[..., 3:] = 0
    ha = [h.clone() for h in a.forward(x)]
    hb = b.forward(x)
    torch.cuda.synchronize()
    assert len(ha) == len(hb) == len(m.LAYER_FACTORS)
    for p, q in zip(ha, hb):
        assert torch.equal(p.view(torch.int16), q.view(torch.int16))


# ------------------------------------------------------------------------------------------------ detector
@pytest.mark.parametrize("name", ['YOLOv4', 'YOLOv4CSP', 'YOLOv4P5', 'YOLOv4Tiny'] + list(ZOO))
def test_every_model_builds_and_detects(name, monkeypatch):
    from fastmot_b200 import YOLODetector
    from fastmot_b200.synth import SyntheticScene
    _synth_env(monkeypatch, name)
    # the aspect filter relaxed as in the end-to-end test: random weights give boxes of any shape
    det = YOLODetector((1920, 1080), [0], model=name, min_aspect_ratio=0.2)
    assert det.backend.n_simt == 0 and len(det.heads) == len(det.model.LAYER_FACTORS)
    dets = det(SyntheticScene(200, seed=3).frame(0))
    assert det.last_num_candidates > 0 and len(dets) > 0
    assert np.all(dets.tlbr[:, 2] >= dets.tlbr[:, 0]) and set(dets.label.tolist()) == {0}


@pytest.mark.parametrize("name", ['YOLOv3Tiny', 'YOLOv4P6'])
def test_yolo_detector_end_to_end_vs_oracle_pipeline(name, monkeypatch):
    """As test_gpu_nets.test_yolo_detector_end_to_end_vs_oracle_pipeline: the detector on a scene frame against the
    oracle pipeline (letterbox geometry, decode, filter_dets) on the same weights.  v3-tiny runs the fp32 oracle conv
    stack (fp16 storage) on the oracle's letterbox.  P6's 200-layer stack turns the last-bit differences of fp16 convs
    summed in another order into score changes that reorder the many near-threshold candidates of synthetic weights,
    so there the oracle decodes the engine's own heads (each launch of that stack is checked against float64 by
    test_zoo_engine_launch_by_launch)."""
    from fastmot_b200 import YOLODetector
    from fastmot_b200.synth import SyntheticScene
    from oracle import nets, detect
    _synth_env(monkeypatch, name)
    frame = SyntheticScene(200, seed=2).frame(0)
    det = YOLODetector((1920, 1080), (0,), name, min_aspect_ratio=0.2)
    got = det(frame)
    m = det.model
    _, H, W = m.INPUT_SHAPE
    roi, up, off = detect.letterbox_geometry((1920, 1080), (W, H), m.LETTERBOX)
    assert (roi, tuple(up), tuple(off)) == (det.roi, tuple(det.upscaled_sz), tuple(det.bbox_offset))
    eng = det.backend
    if name == 'YOLOv4P6':
        heads = [h.permute(2, 0, 1).float().cpu() for h in eng.heads]
    else:
        x = torch.as_tensor(detect.letterbox(frame, (W, H), roi)).half().float()[None]
        weights = {i: (eng.params[i][0].float().cpu().numpy()[..., :3] if i == 0 else
                       eng.params[i][0].float().cpu().numpy(), eng.params[i][1].cpu().numpy()) for i in eng.params}
        with torch.no_grad():
            heads = nets.run_darknet(eng.layers, weights, x, nets.fp16_roundtrip)
    dec = [detect.yolo_decode(h.numpy(), a, s, (W, H), m.NUM_CLASSES, m.NEW_COORDS)
           for h, a, s in zip(heads, m.ANCHORS, m.SCALES)]
    want = detect.filter_dets(np.concatenate(dec), up, off, det.label_mask, 0.25, 0.5, 800000, 0.2)
    assert len(want[0]) > 0
    assert abs(len(got) - len(want[0])) <= max(3, len(want[0]) // 10), (len(got), len(want[0]))
    d = np.abs(got.tlbr[:, None, :] - want[0][None, :, :]).max(-1)
    assert (d.min(1) <= 2).mean() > 0.8


def _per_image_equals_one_image(det, heads, sizes, name):
    """Per image b of det's last detect_batch_async (k = len(sizes) images of those sizes): keys, candidate rows and
    detections bit-identical to the one-image decode + NMS of its head slice with its own size's geometry."""
    from fastmot_b200.detector import YOLODetector
    k, k0, cap = len(sizes), det.num_candidates, det.key_cap
    got = det.postprocess_batch()
    counts = det._counter[:k].cpu().tolist()
    assert all(0 < n <= cap for n in counts), counts
    for b, wh in enumerate(sizes):
        det1 = YOLODetector(wh, (0,), name, engine=NS(heads_nhwc=True))
        det1.postprocess_heads_async([(h[b] if k > 1 else h).contiguous() for h in heads])
        one = det1.postprocess()
        n1 = int(det1._counter.item())
        assert n1 == counts[b], (b, n1, counts[b])
        kb = det._keys[b * cap:b * cap + n1].cpu().numpy().view(np.uint64)
        assert np.array_equal(kb, det1._keys[:n1].cpu().numpy().view(np.uint64)), b
        gidx = (kb & np.uint64(0xffffff)).astype(np.int64)
        rows_b = det._dense[b * k0:(b + 1) * k0].cpu().numpy()[gidx]
        assert np.array_equal(rows_b.view(np.uint32), det1._dense.cpu().numpy()[gidx].view(np.uint32)), b
        assert len(one) > 0
        for f in ('tlbr', 'label', 'conf'):
            assert np.array_equal(got[b][f], one[f]), (b, f)


@pytest.mark.parametrize("name", ['YOLOv3Tiny', 'YOLOv4P6'])
def test_multicamera_step_per_image_equals_one_image_path(name, monkeypatch):
    """A MultiCameraMOT step of a 1080p and a 720p camera (batch 2, per-image geometry), then a step of the 720p camera
    alone (the batch-1 engine that shares the batch-2 one)."""
    from fastmot_b200 import MultiCameraMOT
    from fastmot_b200.synth import SyntheticScene
    from oracle.run import default_tracker_cfg
    _synth_env(monkeypatch, name)
    sizes = [(1920, 1080), (1280, 720)]
    frames = [SyntheticScene(200, size=wh, seed=5 + 7 * s).frame(0) for s, wh in enumerate(sizes)]
    mc = MultiCameraMOT(sizes, detector_frame_skip=5, class_ids=(0,), yolo_detector_cfg=NS(model=name),
                        feature_extractor_cfgs=(NS(model='OSNet025'),), tracker_cfg=NS(**default_tracker_cfg()))
    mc.reset(1 / 30)
    mc.step(frames)
    torch.cuda.synchronize()
    _per_image_equals_one_image(mc.detector, mc.detector.engine(2).heads, sizes, name)
    mc.reset(1 / 30)
    mc.step([None, frames[1]])
    torch.cuda.synchronize()
    assert sorted(mc.detector._engines) == [1, 2]
    _per_image_equals_one_image(mc.detector, mc.detector.engine(1).heads, sizes[1:], name)


@pytest.mark.parametrize("name", ['YOLOv3', 'YOLOv4P6'])
def test_mot_step_schedule_matches_reference_golden(name, monkeypatch):
    """test_gpu_mot.test_mot_step_schedule_matches_reference_golden with this model: the whole detector pipeline runs,
    then the scripted detections replace its rows; the golden schedule's ids and boxes come out."""
    from fastmot_b200 import MOT, DET_DTYPE
    from fastmot_b200.synth import SyntheticScene
    from oracle.run import default_tracker_cfg
    _synth_env(monkeypatch, name)
    g = np.load(os.path.join(GOLDEN, "seq_T64.npz"))
    scene = SyntheticScene(**eval(str(g['scene_kw'])))

    def dets(t):
        tl, lb, cf, _ = scene.detections(t)
        d = np.zeros(len(tl), DET_DTYPE)
        d['tlbr'], d['label'], d['conf'] = tl, lb, cf
        return d.view(np.recarray)

    def embs(t, d):
        return scene.embeddings(scene.detections(t)[3], t)

    mot = MOT(scene.size, detector_frame_skip=5, class_ids=(0,),
              yolo_detector_cfg=NS(model=name), feature_extractor_cfgs=(NS(model='OSNet025'),),
              tracker_cfg=NS(**default_tracker_cfg()), detections_override=dets, embeddings_override=embs)
    assert mot.detector.model.__name__ == name
    mot.reset(1 / 30)
    for t in range(17):
        mot.step(scene.frame(t))
        vis = {trk.trk_id: trk.tlbr for trk in mot.visible_tracks()}
        want = dict(zip(g[f'vis_ids_{t}'].tolist(), g[f'vis_tlbr_{t}']))
        assert set(vis) == set(want), (t, set(vis) ^ set(want))
        for k in vis:
            assert np.abs(vis[k] - want[k]).max() <= 1.0, (t, k)
    assert mot.detector.last_num_candidates > 0
