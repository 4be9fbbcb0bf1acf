"""GPU: cameras of different frame sizes and frame timings in one process (MultiCameraMOT) and the per-frame geometry
kernels under it, on YOLOv4-tiny (no letterbox) and YOLOv4-csp (letterbox; the 4:3 camera gets another ROI).

- Tracking: under a staggered schedule with a dropped frame, a reconnect and an ended camera, every camera holds
  exactly the tracks (ids, boxes bit for bit) a separate MOT of its size holds on that camera's frames alone.
- Per image, the geometry-table letterbox, head decode (+ the unchanged batched NMS) and crops are bit-identical to the
  one-frame entries called with that image's frame and geometry.
- A batch-3 engine sharing a batch-4 engine's memory passes the launch-by-launch float64 check, leaves the 4th image
  alone, gives the heads of a standalone batch-3 engine and allocates (almost) nothing.
"""
import ctypes as C
import time
from types import SimpleNamespace as NS

import numpy as np
import pytest
import torch

from test_gpu_multistream import _boxes, _dets_fn
from test_gpu_yolo_ops import CASES, _bits
from test_multicamera_cpu import schedule

pytestmark = pytest.mark.gpu

SIZES = [(1920, 1080), (1280, 720), (1024, 768)]
MODELS = ['YOLOv4Tiny', 'YOLOv4CSP']


def _synth_env(monkeypatch, name):
    """build_yolo_engine's synthetic heads at test_gpu_yolo_ops.py's bias / gain: a few hundred to ~1500 candidates
    per frame, inside key_cap."""
    bias, gain, _ = CASES[name]
    monkeypatch.setenv("FM_SYNTH_OBJ_BIAS", str(bias))
    monkeypatch.setenv("FM_SYNTH_HEAD_GAIN", str(gain))


def _nets_kw(name):
    from oracle.run import default_tracker_cfg
    return dict(detector_frame_skip=5, class_ids=(0,), yolo_detector_cfg=NS(model=name),
                feature_extractor_cfgs=(NS(model='OSNet025'),), tracker_cfg=NS(**default_tracker_cfg()))


# ------------------------------------------------------------------------------------------------ tracking
@pytest.mark.parametrize("name", MODELS)
def test_multicamera_tracks_equal_separate_mot_per_camera(name, monkeypatch):
    """The schedule of test_multicamera_cpu.schedule (batches of k = 1, 2 and 3): each camera against separate MOTs
    of its size fed only its frames, a fresh MOT after camera 1's reconnect."""
    from fastmot_b200 import MOT, MultiCameraMOT
    from fastmot_b200.synth import SyntheticScene
    _synth_env(monkeypatch, name)
    plans = schedule()
    T = len(plans)
    present = [[s in sum(p, []) for s in range(3)] for p in plans]
    scenes = [SyntheticScene(64, size=wh, seed=3 + 101 * s) for s, wh in enumerate(SIZES)]
    dets = [_dets_fn(sc) for sc in scenes]
    frames = [[sc.frame(t) if present[t][s] else None for s, sc in enumerate(scenes)] for t in range(T)]
    # segments: the steps each camera's consecutive local frames come from (camera 1 restarts at step 14)
    segs = [[[t for t in range(T) if present[t][s]]] for s in range(3)]
    segs[1] = [[t for t in segs[1][0] if t < 14], [t for t in segs[1][0] if t >= 14]]

    def emb(s, t):
        return scenes[s].embeddings(scenes[s].detections(t)[3], t)

    want = [[{}] * T for _ in range(3)]             # visible tracks after step t; kept while the camera is absent
    for s in range(3):
        for j, seg in enumerate(segs[s]):
            end = segs[s][j + 1][0] if j + 1 < len(segs[s]) else T
            mot = MOT(SIZES[s], detections_override=lambda i, seg=seg, s=s: dets[s](seg[i]),
                      embeddings_override=lambda i, d, seg=seg, s=s: emb(s, seg[i]), **_nets_kw(name))
            mot.reset(1 / 30)
            vis = {}
            for t in range(seg[0], end):
                if t in seg:
                    mot.step(frames[t][s])
                    vis = {trk.trk_id: trk.tlbr.copy() for trk in mot.visible_tracks()}
                want[s][t] = vis
            del mot

    cur = [segs[s][0] for s in range(3)]
    mc = MultiCameraMOT(SIZES, detections_override=lambda s, i: dets[s](cur[s][i]),
                        embeddings_override=lambda s, i, d: emb(s, cur[s][i]), **_nets_kw(name))
    mc.reset(1 / 30)
    ks = set()
    for t in range(T):
        if t == 14:
            mc.reset_stream(1, 1 / 30)
            cur[1] = segs[1][1]
        mc.step(frames[t])
        k = len(plans[t][0]) + len(plans[t][1])
        if k:
            ks.add(k)
            assert len(mc.detector.last_num_candidates) == k, t
        for s in range(3):
            assert mc.frame_counts[s] == sum(1 for u in cur[s] if u <= t), (t, s)
            vis = {trk.trk_id: trk.tlbr for trk in mc.visible_tracks(s)}
            assert set(vis) == set(want[s][t]), (s, t, set(vis) ^ set(want[s][t]))
            for i in vis:
                assert np.array_equal(vis[i], want[s][t][i]), (s, t, i)
    assert ks == {1, 2, 3}
    assert sorted(mc.detector._engines) == [1, 2, 3]
    assert any(want[s][T - 1] for s in range(3))


def test_multicamera_overflow_names_the_camera(monkeypatch):
    """max_dets overflow on camera 2 while it is slot 0 of the step's batch: the error names camera 2."""
    from fastmot_b200 import MultiCameraMOT
    from fastmot_b200.synth import SyntheticScene
    _synth_env(monkeypatch, 'YOLOv4Tiny')
    kw = _nets_kw('YOLOv4Tiny')
    kw['yolo_detector_cfg'] = NS(model='YOLOv4Tiny', max_dets=1)
    mc = MultiCameraMOT(SIZES, **kw)
    mc.reset(1 / 30)
    f2 = SyntheticScene(200, size=SIZES[2], seed=9).frame(0)
    with pytest.raises(RuntimeError, match="camera 2: more than max_dets"):
        mc.step([None, None, f2])


# ------------------------------------------------------------------------------------------------ kernels
class GeomCase:
    """A batch-4 engine with test_gpu_yolo_ops.py's synthetic weights and its detector, run on three frames of the
    three sizes: detect_batch_async builds the batch-3 engine that shares the batch-4 one (without a graph) and
    records how much device memory that took.  The batch-4 engine itself never runs, so the 4th image of each of its
    buffers holds the zeros it was allocated with unless the batch-3 engine writes there."""

    def __init__(self, name):
        from fastmot_b200 import models
        from fastmot_b200.detector import YOLODetector
        from fastmot_b200.engine import YoloEngine
        from fastmot_b200.models import darknet
        from fastmot_b200.synth import SyntheticScene
        bias, gain, _ = CASES[name]
        self.name = name
        m = self.model = models.YOLO.get_model(name)
        self.layers = darknet.BUILDERS[m.CFG](num_classes=m.NUM_CLASSES, anchors_per_head=len(m.ANCHORS[0]) // 2)
        self.weights = darknet.synthetic_weights(self.layers, 3, head_obj_bias=bias, num_classes=m.NUM_CLASSES,
                                                 head_gain=gain)
        self.eng4 = YoloEngine(self.layers, m.INPUT_SHAPE[1:], self.weights, use_graph=False, batch=4)
        self.classes = tuple(range(m.NUM_CLASSES))
        self.det = YOLODetector(SIZES[0], self.classes, name, engine=self.eng4, batch=4)
        self.frames = [torch.as_tensor(SyntheticScene(200, size=wh, seed=5 + 7 * b).frame(b)).cuda()
                       for b, wh in enumerate(SIZES)]
        torch.cuda.synchronize()
        base = torch.cuda.memory_allocated()
        self.eng3 = self.det.engine(3)
        torch.cuda.synchronize()
        self.grew = torch.cuda.memory_allocated() - base
        self.fourth = [t[3].clone() for t in self.eng4._bufs]
        self.det.detect_batch_async(self.frames)
        self.got = self.det.postprocess_batch()
        torch.cuda.synchronize()

    def close(self):
        self.eng3 = self.eng4 = self.det = None
        torch.cuda.empty_cache()


@pytest.fixture(scope="module", params=MODELS)
def gcase(request):
    c = GeomCase(request.param)
    yield c
    c.close()


def test_geom_letterbox_equals_fmframe_letterbox(gcase):
    from fastmot_b200 import _lib
    from fastmot_b200.devmem import Frame, ptr, stream_ptr
    det = gcase.det
    lib = _lib.load()
    rois = [det.geometry(wh)[0] for wh in SIZES]
    if gcase.model.LETTERBOX:
        assert rois[0] == rois[1] != rois[2], rois
    for b, (f, wh) in enumerate(zip(gcase.frames, SIZES)):
        rx, ry, rw, rh = rois[b]
        one = torch.zeros_like(det.inp[0])
        fm = Frame.bgr(f).fm()
        assert (fm.w, fm.h) == wh
        _lib.check(lib.fm_letterbox_preproc(C.byref(fm), det.input_wh[0], det.input_wh[1], rx, ry, rw, rh, 1, ptr(one),
                                            stream_ptr()), "fm_letterbox_preproc")
        torch.cuda.synchronize()
        assert torch.equal(det.inp[b].view(torch.int16), one.view(torch.int16)), (gcase.name, b)


def test_geom_decode_and_nms_equal_one_image_path(gcase):
    """Per image of the batch-3 detection: sorted keys, dense rows and detections equal the one-image decode + NMS of
    its head slice with its own size's geometry, bit for bit; the detections equal filter_dets on its candidates."""
    from oracle import detect
    from fastmot_b200.detector import YOLODetector
    det, k0, cap = gcase.det, gcase.det.num_candidates, gcase.det.key_cap
    det.postprocess_heads_batch_async(gcase.eng3.heads, 3, det._geom)
    got = det.postprocess_batch()
    counts = det._counter[:3].cpu().tolist()
    assert all(0 < n <= cap for n in counts), counts
    for b, wh in enumerate(SIZES):
        assert np.array_equal(got[b].tlbr, gcase.got[b].tlbr)
        det1 = YOLODetector(wh, gcase.classes, gcase.name, engine=NS(heads_nhwc=True))
        det1.postprocess_heads_async([h[b].contiguous() for h in gcase.eng3.heads])
        one = det1.postprocess()
        n1 = int(det1._counter.item())
        assert n1 == counts[b], (b, n1, counts[b])
        kb = det._keys[b * cap:b * cap + n1].cpu().numpy().view(np.uint64)
        assert np.array_equal(kb, det1._keys[:n1].cpu().numpy().view(np.uint64)), b
        gidx = (kb & np.uint64(0xffffff)).astype(np.int64)
        rows_b = det._dense[b * k0:(b + 1) * k0].cpu().numpy()[gidx]
        assert np.array_equal(rows_b.view(np.uint32), det1._dense.cpu().numpy()[gidx].view(np.uint32)), b
        for f in ('tlbr', 'label', 'conf'):
            assert np.array_equal(got[b][f], one[f]), (b, f)
        want = detect.filter_dets(rows_b[np.argsort(gidx), :7], (1.0, 1.0), (0.0, 0.0), det.label_mask,
                                  det.conf_thresh, det.nms_thresh, det.max_area, det.min_aspect_ratio)
        assert len(got[b]) == len(want[0]) > 0
        assert np.array_equal(got[b].tlbr, want[0]) and np.array_equal(got[b].label, want[1])
        assert np.array_equal(got[b].conf, want[2])


def test_geom_crops_equal_fmframe_crops():
    """Mixed-size crops, including boxes past the right and bottom edges of the smaller frames, equal
    fm_roi_resize_norm on their own frame bit for bit."""
    from fastmot_b200 import _lib
    from fastmot_b200.devmem import Frame, ptr, stream_ptr
    from fastmot_b200.feature_extractor import FeatureExtractor
    from fastmot_b200.synth import SyntheticScene
    lib = _lib.load()
    frames = [torch.as_tensor(SyntheticScene(100, size=wh, seed=40 + s).frame(s)).cuda() for s, wh in enumerate(SIZES)]
    boxes = []
    for s, (w, h) in enumerate(SIZES):
        b = _boxes(37, 60 + s) * np.array([w / 1920, h / 1080] * 2)
        edge = np.array([[w - 40.5, h - 90.2, w + 55.0, h + 30.0], [w - 1.0, 10.0, w + 300.0, 200.0],
                         [5.0, h - 2.0, 120.0, h + 400.0]])
        boxes.append(np.concatenate([b, edge]))
    fe = FeatureExtractor('OSNet025', max_crops=sum(len(b) for b in boxes), use_graph=False)
    fe.extract_multi_async(frames, boxes)
    outs = fe.postprocess()
    torch.cuda.synchronize()
    eng = fe._engine(sum(len(b) for b in boxes))
    assert [len(o) for o in outs] == [len(b) for b in boxes]
    r0 = 0
    for s, (w, h) in enumerate(SIZES):
        n = len(boxes[s])
        one = torch.zeros_like(eng.inp[:n])
        tl = torch.as_tensor(boxes[s]).cuda()
        fm = Frame.bgr(frames[s]).fm()
        assert (fm.w, fm.h) == (w, h)
        _lib.check(lib.fm_roi_resize_norm(C.byref(fm), ptr(tl), None, n, 128, 256, eng.inp_layout, ptr(one),
                                          stream_ptr()), "fm_roi_resize_norm")
        torch.cuda.synchronize()
        assert torch.equal(eng.inp[r0:r0 + n].view(torch.int16), one.view(torch.int16)), s
        r0 += n


def test_shared_engine_launch_by_launch_heads_and_memory(gcase, monkeypatch):
    """The batch-3 engine that shares the batch-4 engine: test_gpu_yolo_ops.run_launch_by_launch over its 3 images
    (inputs bit for bit, nothing written outside the output views, outputs within the float64 bound), the 4th image
    of every shared buffer untouched, heads bit-identical to a standalone batch-3 engine with the same weights, and
    less than 1 % of the batch-4 engine's buffer bytes allocated to build it."""
    import test_gpu_yolo_ops as Y
    from fastmot_b200.engine import YoloEngine
    eng3, eng4 = gcase.eng3, gcase.eng4
    buf_bytes = sum(t.numel() * t.element_size() for t in eng4._bufs)
    assert gcase.grew < 0.01 * buf_bytes, (gcase.grew, buf_bytes)
    assert all(a.data_ptr() == b.data_ptr() for a, b in zip(eng3._bufs, eng4._bufs))
    assert all(eng3.params[i][0].data_ptr() == eng4.params[i][0].data_ptr() for i in eng4.params)
    assert eng3.ws.data_ptr() == eng4.ws.data_ptr()
    assert len(eng3.launches) == len(eng4.launches) == len(eng3.trace)

    def region(v, t):
        return t.reshape(-1)[:3 * v.h * v.w * v.c_stride].view(3, v.h, v.w, v.c_stride)[..., v.c_off:v.c_off + v.c]

    def first_diff(a, b):
        i = int((_bits(a) != _bits(b)).reshape(-1).nonzero()[0])
        return tuple(int(x) for x in np.unravel_index(i, a.shape))

    monkeypatch.setattr(Y, "_region", region)
    monkeypatch.setattr(Y, "_first_diff", first_diff)
    t0 = time.time()
    worst = Y.run_launch_by_launch(eng3, f"{gcase.name} shared k=3 of 4")
    print(f"\n[multicamera yolo ops] {gcase.name} k=3 of 4: {len(eng3.trace)} launches, {time.time() - t0:.1f} s; " +
          ", ".join(f"{k}{'/' + p if p else ''} {v:.3f}" for (k, p), v in sorted(worst.items(), key=str)))
    for i, (t, was) in enumerate(zip(eng4._bufs, gcase.fourth)):
        assert torch.equal(t[3].view(torch.int16), was.view(torch.int16)), f"buffer {i}: image 3 written"

    alone = YoloEngine(gcase.layers, gcase.model.INPUT_SHAPE[1:], gcase.weights, use_graph=False, batch=3)
    alone.forward(gcase.det.inp[:3])
    eng3.forward(gcase.det.inp[:3])
    torch.cuda.synchronize()
    for a, b in zip(eng3.heads, alone.heads):
        assert a.shape == b.shape
        assert torch.equal(_bits(a), _bits(b))


@pytest.mark.parametrize("name", MODELS)
def test_detector_size_frames_run_the_batch_b_engine(name, monkeypatch):
    """B = 2 different frames of the detector's own size through detect_batch_async: the batch-2 engine runs them (no
    batch-k engine is built), each image's letterbox equals fm_letterbox_preproc on its frame bit for bit, and each
    image's keys, candidate rows and detections equal the one-image decode + NMS of its head slice."""
    from test_gpu_yolo_zoo import _per_image_equals_one_image
    from fastmot_b200 import _lib
    from fastmot_b200.detector import YOLODetector
    from fastmot_b200.devmem import Frame, ptr, stream_ptr
    from fastmot_b200.synth import SyntheticScene
    _synth_env(monkeypatch, name)
    size = SIZES[0]
    det = YOLODetector(size, (0,), name, batch=2)
    frames = [torch.as_tensor(SyntheticScene(200, size=size, seed=5 + 7 * b).frame(b)).cuda() for b in range(2)]
    det.detect_batch_async(frames)
    torch.cuda.synchronize()
    assert sorted(det._engines) == [2]
    lib = _lib.load()
    rx, ry, rw, rh = det.roi
    for b, f in enumerate(frames):
        one = torch.zeros_like(det.inp[0])
        fm = Frame.bgr(f).fm()
        assert (fm.w, fm.h) == tuple(size)
        _lib.check(lib.fm_letterbox_preproc(C.byref(fm), det.input_wh[0], det.input_wh[1], rx, ry, rw, rh, 1, ptr(one),
                                            stream_ptr()), "fm_letterbox_preproc")
        torch.cuda.synchronize()
        assert torch.equal(det.inp[b].view(torch.int16), one.view(torch.int16)), (name, b)
    assert not torch.equal(det.inp[0], det.inp[1])
    _per_image_equals_one_image(det, det.backend.heads, [size] * 2, name)
