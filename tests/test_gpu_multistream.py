"""GPU: several camera streams in one process (MultiStreamMOT) and the batched kernels under it.

- Tracking: every stream of a MultiStreamMOT holds exactly the tracks (ids, boxes bit for bit) a separate MOT holds
  on that stream alone; two MOT objects in one process number their own tracks.
- Batched detector, per image: the batched letterbox equals the one-frame letterbox bit for bit; every launch of a
  B = 4 engine is checked alone against oracle/nets64.py (as tests/test_gpu_yolo_ops.py does at B = 1); each image's
  candidate table and detections equal the one-image decode + NMS of its head slice; NMS never crosses images.
- Shared ReID batch: the multi-frame crops equal the one-frame crops bit for bit; the shared forward's per-stream
  embeddings agree with per-stream forwards, and its launches pass the float64 check at 3 x 67 crops.
"""
import ctypes as C
import os
import time
from types import SimpleNamespace as NS

import numpy as np
import pytest
import torch

from conftest import GOLDEN

pytestmark = pytest.mark.gpu

B = 4


def _dets_fn(scene):
    from fastmot_b200 import DET_DTYPE

    def dets(t):
        tl, lb, cf, _ = scene.detections(t)
        d = np.zeros(len(tl), DET_DTYPE)
        d['tlbr'], d['label'], d['conf'] = tl, lb, cf
        return d.view(np.recarray)
    return dets


def _nets_kw():
    from oracle.run import default_tracker_cfg
    return dict(detector_frame_skip=5, class_ids=(0,), yolo_detector_cfg=NS(model='YOLOv4Tiny'),
                feature_extractor_cfgs=(NS(model='OSNet025'),), tracker_cfg=NS(**default_tracker_cfg()))


# ------------------------------------------------------------------------------------------------ tracking
def test_multistream_tracks_equal_separate_mot_per_stream():
    from fastmot_b200 import MOT, MultiStreamMOT
    from fastmot_b200.synth import SyntheticScene
    g = np.load(os.path.join(GOLDEN, "seq_T64.npz"))
    kw = eval(str(g['scene_kw']))
    scenes = [SyntheticScene(**kw), SyntheticScene(**dict(kw, seed=kw.get('seed', 0) + 101)),
              SyntheticScene(**dict(kw, seed=kw.get('seed', 0) + 202))]
    dets = [_dets_fn(s) for s in scenes]
    T = 18
    frames = [[s.frame(t) for s in scenes] for t in range(T)]

    def embs(s):
        return lambda t, d: scenes[s].embeddings(scenes[s].detections(t)[3], t)

    want = []
    for s in range(3):
        mot = MOT(scenes[s].size, detections_override=dets[s], embeddings_override=embs(s), **_nets_kw())
        mot.reset(1 / 30)
        seq = []
        for t in range(T):
            mot.step(frames[t][s])
            seq.append({trk.trk_id: trk.tlbr.copy() for trk in mot.visible_tracks()})
        want.append(seq)

    ms = MultiStreamMOT(scenes[0].size, 3, detections_override=lambda s, t: dets[s](t),
                        embeddings_override=lambda s, t, d: embs(s)(t, d), **_nets_kw())
    ms.reset(1 / 30)
    for t in range(T):
        ms.step(frames[t])
        assert ms.frame_count == t + 1
        for s in range(3):
            vis = {trk.trk_id: trk.tlbr for trk in ms.visible_tracks(s)}
            assert set(vis) == set(want[s][t]), (s, t, set(vis) ^ set(want[s][t]))
            for k in vis:
                assert np.array_equal(vis[k], want[s][t][k]), (s, t, k)
        gw = dict(zip(g[f'vis_ids_{t}'].tolist(), g[f'vis_tlbr_{t}']))
        vis0 = {trk.trk_id: trk.tlbr for trk in ms.visible_tracks(0)}
        assert set(vis0) == set(gw), (t, set(vis0) ^ set(gw))
        for k in vis0:
            assert np.abs(vis0[k] - gw[k]).max() <= 1.0, (t, k)
    assert len(ms.detector.last_num_candidates) == 3
    ms.reset(1 / 30)
    ms.step(frames[0])
    for s in range(3):
        ids = sorted(trk.trk_id for trk in ms.trackers[s].tracks.values())
        assert ids == list(range(1, len(dets[s](0)) + 1)), (s, ids[:5])


def test_two_mot_objects_number_their_own_tracks():
    """Two MOT objects stepped alternately in one process: each numbers its tracks from 1."""
    from fastmot_b200 import MOT
    from fastmot_b200.synth import SyntheticScene
    scenes = [SyntheticScene(30, seed=5, label=0, dropout_frames=()), SyntheticScene(20, seed=6, label=0,
                                                                                     dropout_frames=())]
    mots = [MOT(s.size, detections_override=_dets_fn(s), **_nets_kw()) for s in scenes]
    for m in mots:
        m.reset(1 / 30)
    for t in range(2):
        for m, s in zip(mots, scenes):
            m.step(s.frame(t))
            assert sorted(m.tracker.tracks) == list(range(1, len(s.detections(0)[0]) + 1)), t
    mots[0].reset(1 / 30)
    mots[0].step(scenes[0].frame(0))
    assert min(mots[0].tracker.tracks) == 1
    assert sorted(mots[1].tracker.tracks) == list(range(1, len(scenes[1].detections(0)[0]) + 1))


def test_multistream_rejects_out_of_scope_settings():
    from fastmot_b200 import MultiStreamMOT
    with pytest.raises(NotImplementedError):
        MultiStreamMOT((1920, 1080), 2, detector_type='PUBLIC')
    with pytest.raises(NotImplementedError):
        MultiStreamMOT((1920, 1080), 2, detector_type='SSD')
    with pytest.raises(ValueError):
        MultiStreamMOT([(1920, 1080), (1280, 720)], 2)


# ------------------------------------------------------------------------------------------------ batched detector
class BatchCase:
    """A B = 4 engine with test_gpu_yolo_ops.py's synthetic weights, its detector, four different frames through the
    batched letterbox, and a one-image detector sharing nothing but the decode / NMS settings."""

    def __init__(self, name):
        from test_gpu_yolo_ops import CASES
        from fastmot_b200 import models
        from fastmot_b200.detector import YOLODetector
        from fastmot_b200.engine import YoloEngine
        from fastmot_b200.models import darknet
        from fastmot_b200.synth import SyntheticScene
        bias, gain, _ = CASES[name]
        self.name = name
        m = self.model = models.YOLO.get_model(name)
        layers = darknet.BUILDERS[m.CFG](num_classes=m.NUM_CLASSES, anchors_per_head=len(m.ANCHORS[0]) // 2)
        weights = darknet.synthetic_weights(layers, 3, head_obj_bias=bias, num_classes=m.NUM_CLASSES, head_gain=gain)
        self.eng = YoloEngine(layers, m.INPUT_SHAPE[1:], weights, use_graph=False, batch=B)
        classes = tuple(range(m.NUM_CLASSES))
        self.det = YOLODetector((1920, 1080), classes, name, engine=self.eng, batch=B)
        self.det1 = YOLODetector((1920, 1080), classes, name, engine=NS(heads_nhwc=True))
        self.frames = [torch.as_tensor(SyntheticScene(200, seed=3 + 7 * b).frame(b)).cuda() for b in range(B)]
        self.det.preprocess_frames(self.frames)
        self.eng.forward(self.det.inp)
        torch.cuda.synchronize()

    def close(self):
        self.eng = self.det = self.det1 = None
        torch.cuda.empty_cache()


# plain resize with old head coordinates (tiny-416, YOLOv4-512) and letterbox with new ones (csp-640, P5-896)
@pytest.fixture(scope="module", params=['YOLOv4Tiny', 'YOLOv4CSP', 'YOLOv4', 'YOLOv4P5'])
def bcase(request):
    c = BatchCase(request.param)
    yield c
    c.close()


def test_batched_letterbox_equals_fmframe_letterbox(bcase):
    from fastmot_b200 import _lib
    from fastmot_b200.devmem import Frame, ptr, stream_ptr
    det = bcase.det
    lib = _lib.load()
    rx, ry, rw, rh = det.roi
    for b, f in enumerate(bcase.frames):
        one = torch.zeros_like(det.inp[0])
        fm = Frame.bgr(f).fm()
        assert (fm.w, fm.h) == (1920, 1080)
        _lib.check(lib.fm_letterbox_preproc(C.byref(fm), det.input_wh[0], det.input_wh[1], rx, ry, rw, rh, 1, ptr(one),
                                            stream_ptr()), "fm_letterbox_preproc")
        torch.cuda.synchronize()
        assert torch.equal(det.inp[b].view(torch.int16), one.view(torch.int16)), b
    assert not torch.equal(det.inp[0], det.inp[1])


def _region_b(v, t):
    """View v's elements in tensor t (a buffer of v's shape: [B][h][w][c_stride] fp16) as (B, h, w, c)."""
    return t.reshape(-1)[:B * v.h * v.w * v.c_stride].view(B, v.h, v.w, v.c_stride)[..., v.c_off:v.c_off + v.c]


def _first_diff_b(a, b):
    from test_gpu_yolo_ops import _bits
    i = int((_bits(a) != _bits(b)).reshape(-1).nonzero()[0])
    return tuple(int(x) for x in np.unravel_index(i, a.shape))


def test_batched_engine_launch_by_launch(bcase):
    """test_gpu_yolo_ops.run_launch_by_launch at B = 4: inputs bit for bit, nothing written outside the output view,
    every output element of every image within the float64 reference's bound.  The 1x1 convs that stay on conv_tma
    flatten n * ho * wo into one row dimension; the 3x3 ones move to conv_tc at n > 1."""
    from test_gpu_yolo_ops import _bits, _reference_ratio
    from fastmot_b200.devmem import stream_ptr
    eng = bcase.eng
    t0 = time.time()
    paths = {(e.kind, e.info.get('path'), eng.layers[e.ops[0]].get('size')) for e in eng.trace if 'path' in e.info}
    assert ('conv', 'tma', 1) in paths, paths
    assert not any(p == 'tma' and k == 3 for _, p, k in paths), paths
    assert len(eng.trace) == len(eng.launches)
    last = {}
    for k, e in enumerate(eng.trace):
        for v in e.ins + e.outs:
            last[v.t.data_ptr()] = k
    shadow = {eng.inp.data_ptr(): eng.inp.clone()}
    written = {eng.inp.data_ptr(): torch.ones(eng.inp.shape[-1], dtype=torch.bool)}
    worst = {}
    sp = stream_ptr()
    torch.cuda.synchronize()
    for k, e in enumerate(eng.trace):
        path = e.info.get('path')
        where = f"{bcase.name} B={B}: launch {k} ({e.kind}{'/' + path if path else ''}, layers {list(e.ops)})"
        ins = []
        for v in e.ins:
            p = v.t.data_ptr()
            assert p in written and bool(written[p][v.c_off:v.c_off + v.c].all()), (where, v.name)
            was, now = _region_b(v, shadow[p]), _region_b(v, v.t)
            if not torch.equal(_bits(now), _bits(was)):
                pytest.fail(f"{where}: input '{v.name}' overwritten, first at b/y/x/ch {_first_diff_b(now, was)}")
            ins.append(was)
        before = {v.t.data_ptr(): v.t.clone() for v in e.outs}
        eng.launches[k](sp)
        torch.cuda.synchronize()
        for v in e.outs:
            p = v.t.data_ptr()
            after = v.t.clone()
            a, b = after.reshape(-1, v.c_stride), before[p].reshape(-1, v.c_stride)
            for sl in (slice(0, v.c_off), slice(v.c_off + v.c, v.c_stride)):
                if not torch.equal(_bits(a[:, sl]), _bits(b[:, sl])):
                    pytest.fail(f"{where}: wrote outside its view '{v.name}'")
            shadow[p] = after
            written.setdefault(p, torch.zeros(v.c_stride, dtype=torch.bool))[v.c_off:v.c_off + v.c] = True
        o = e.outs[0]
        got = _region_b(o, shadow[o.t.data_ptr()])
        r = _reference_ratio(eng, e, ins, got, f"{where}: output '{o.name}'")
        worst[(e.kind, path)] = max(worst.get((e.kind, path), 0.0), r)
        for p in [p for p, j in last.items() if j == k]:
            shadow.pop(p, None)
    print(f"\n[multistream yolo ops] {bcase.name} B={B}: {len(eng.trace)} launches, {time.time() - t0:.1f} s; " +
          ", ".join(f"{k}{'/' + p if p else ''} {v:.3f}" for (k, p), v in sorted(worst.items(), key=str)))


def _sorted_keys(keys_dev, n):
    return keys_dev[:n].cpu().numpy().view(np.uint64)


def test_batched_decode_and_nms_equal_one_image_path(bcase):
    """Per image: the sorted key table, the dense rows and the detections of the batched decode + NMS equal the
    one-image decode + NMS of that image's head slice bit for bit; the detections equal filter_dets on the image's own
    candidates."""
    from oracle import detect
    det, det1, k0, cap = bcase.det, bcase.det1, bcase.det.num_candidates, bcase.det.key_cap
    det.postprocess_heads_batch_async(bcase.eng.heads)
    got = det.postprocess_batch()
    counts = det._counter.cpu().tolist()
    assert all(20 <= n <= cap // 2 for n in counts), counts
    for b in range(B):
        det1.postprocess_heads_async([h[b].contiguous() for h in bcase.eng.heads])
        one = det1.postprocess()
        n1 = int(det1._counter.item())
        assert n1 == counts[b], (b, n1, counts[b])
        kb = _sorted_keys(det._keys[b * cap:], n1)
        assert np.array_equal(kb, _sorted_keys(det1._keys, n1)), b
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


def test_batched_detector_empty_image_and_max_dets_overflow_names_the_image(bcase):
    """An image whose heads hold no candidate gives no detection; an image with more survivors than max_dets raises
    and the message names it."""
    from fastmot_b200.detector import YOLODetector
    m = bcase.model
    heads = [h.clone() for h in bcase.eng.heads]
    for h in heads:                                  # objectness 0 (after the sigmoid of old-coords heads)
        h[0] = -30.0 if not m.NEW_COORDS else 0.0
    det = bcase.det
    det.postprocess_heads_batch_async(heads)
    got = det.postprocess_batch()
    assert det.last_num_candidates[0] == 0 and len(got[0]) == 0
    assert all(len(g) > 0 for g in got[1:])
    small = YOLODetector((1920, 1080), tuple(range(m.NUM_CLASSES)), bcase.name, engine=NS(heads_nhwc=True, batch=B),
                         batch=B, max_dets=len(got[2]) - 1)
    for h in heads:
        for b in (1, 3):
            h[b] = h[0]
    small.postprocess_heads_batch_async(heads)
    with pytest.raises(RuntimeError, match="image 2: more than max_dets"):
        small.postprocess_batch()


def test_batched_nms_never_suppresses_across_images():
    """fm_diou_nms_filter_batch on hand-made tables: image 0 empty, images 1 and 2 identical (each keeps exactly what
    filter_dets keeps on it alone), image 3 over max_out (status 2 for image 3 only)."""
    from test_gpu_yolo_ops import _nms_table
    from oracle import detect
    from fastmot_b200 import _lib
    from fastmot_b200.devmem import ptr, stream_ptr
    lib = _lib.load()
    cap = stride = 4096
    tables = [None, _nms_table(2049, seed=11), _nms_table(2049, seed=11), _nms_table(4096, seed=12)]
    wants = [None] + [detect.filter_dets(t[0][:, :7], (1.0, 1.0), (0.0, 0.0), np.ones(2, bool), 0.0, 0.5, 12000.0, 0.8)
                      for t in tables[1:]]
    max_out = len(wants[1][0])                       # images 1 and 2 fit exactly, image 3 has more survivors
    assert len(wants[3][0]) > max_out
    keys = torch.zeros(B * cap, dtype=torch.int64, device="cuda")
    dense = torch.zeros(B * stride, 8, dtype=torch.float32, device="cuda")
    counters = torch.zeros(B, dtype=torch.int32, device="cuda")
    for b, tb in enumerate(tables):
        if tb is None:
            continue
        rows, k = tb
        keys[b * cap:b * cap + len(k)] = torch.as_tensor(k.view(np.int64)).cuda()
        dense[b * stride:b * stride + len(rows)] = torch.as_tensor(rows).cuda()
        counters[b] = len(k)
    mask = torch.zeros(B * int(lib.fm_nms_mask_bytes(cap)), dtype=torch.uint8, device="cuda")
    o_t = torch.zeros(B * max_out, 4, dtype=torch.float64, device="cuda")
    o_l = torch.zeros(B * max_out, dtype=torch.int64, device="cuda")
    o_c = torch.zeros(B * max_out, dtype=torch.float64, device="cuda")
    cnt = torch.zeros(B, dtype=torch.int32, device="cuda")
    st = torch.full((B,), 7, dtype=torch.int32, device="cuda")
    _lib.check(lib.fm_diou_nms_filter_batch(B, ptr(keys), ptr(dense), stride, ptr(counters), cap, 0.5, 12000.0, 0.8,
                                            ptr(mask), max_out, ptr(o_t), ptr(o_l), ptr(o_c), ptr(cnt), ptr(st),
                                            stream_ptr()), "fm_diou_nms_filter_batch")
    torch.cuda.synchronize()
    cnt, st = cnt.cpu().tolist(), st.cpu().tolist()
    assert st == [0, 0, 0, 2], st
    assert cnt[0] == 0 and cnt[3] == max_out
    for b in (1, 2, 3):
        want = wants[b]
        n = cnt[b]
        assert n == min(len(want[0]), max_out), (b, n, len(want[0]))
        sl = slice(b * max_out, b * max_out + n)
        assert np.array_equal(o_t.cpu().numpy()[sl], want[0][:n]), b
        assert np.array_equal(o_l.cpu().numpy()[sl], want[1][:n]), b
        assert np.array_equal(o_c.cpu().numpy()[sl], want[2][:n]), b


# ------------------------------------------------------------------------------------------------ shared ReID batch
def _boxes(n, seed):
    rng = np.random.default_rng(seed)
    x0 = rng.uniform(-20, 1800, n)
    y0 = rng.uniform(-20, 900, n)
    w = rng.uniform(8, 300, n)
    h = w * rng.uniform(1.0, 3.0, n)
    return np.stack([x0, y0, x0 + w, y0 + h], 1)


def test_shared_reid_batch_equals_fmframe_crops():
    """3 streams x 67 crops (201, not a multiple of 8): every crop of fm_roi_resize_norm_geom equals the one-frame
    crop bit for bit; the shared forward's per-stream rows agree with one forward per stream (<= 5e-3 abs) and are
    views of the shared output; every launch of the shared forward passes the float64 check."""
    from test_gpu_osnet_ops import run_launch_by_launch
    from fastmot_b200 import _lib
    from fastmot_b200.devmem import Frame, ptr, stream_ptr
    from fastmot_b200.feature_extractor import FeatureExtractor
    from fastmot_b200.synth import SyntheticScene
    from fastmot_b200.tracker import DeviceEmbeddings
    lib = _lib.load()
    S, n = 3, 67
    frames = [torch.as_tensor(SyntheticScene(100, seed=40 + s).frame(s)).cuda() for s in range(S)]
    boxes = [_boxes(n, 50 + s) for s in range(S)]
    fe = FeatureExtractor('OSNet10', max_crops=S * n, use_graph=False)
    fe.extract_multi_async(frames, boxes)
    outs = fe.postprocess()
    torch.cuda.synchronize()
    eng = fe._engine(S * n)
    assert eng.max_batch == 208
    shared = eng.inp[:S * n].clone()
    for s in range(S):                                   # the crops, bit for bit
        one = torch.zeros_like(eng.inp[:n])
        tl = torch.as_tensor(boxes[s]).cuda()
        fm = Frame.bgr(frames[s]).fm()
        assert (fm.w, fm.h) == (1920, 1080)
        _lib.check(lib.fm_roi_resize_norm(C.byref(fm), ptr(tl), None, n, 128, 256, eng.inp_layout, ptr(one),
                                          stream_ptr()), "fm_roi_resize_norm")
        torch.cuda.synchronize()
        assert torch.equal(shared[s * n:(s + 1) * n].view(torch.int16), one.view(torch.int16)), s
    assert len(outs) == S and all(isinstance(o, DeviceEmbeddings) and len(o) == n for o in outs)
    base = eng.out.data_ptr()
    for s, o in enumerate(outs):                         # views into the shared output
        assert o.tensor.data_ptr() == base + s * n * eng.out.shape[1] * 4
    got = [np.asarray(o).copy() for o in outs]
    for s in range(S):                                   # one forward per stream
        fe1 = FeatureExtractor('OSNet10', max_crops=n, use_graph=False)
        fe1.extract_async(frames[s], boxes[s])
        want = np.asarray(fe1.postprocess())
        assert np.abs(got[s] - want).max() <= 5e-3, (s, float(np.abs(got[s] - want).max()))
    fe.extract_multi_async(frames, boxes)               # every launch of the shared forward alone
    torch.cuda.synchronize()
    crops = torch.zeros(eng.max_batch, 256, 128, 8, dtype=torch.float16, device="cuda")
    crops[..., :3] = eng.inp[:, 4:-4, 4:-4, :3] if eng.inp_layout == 2 else eng.inp[..., :3]
    t0 = time.time()
    worst = run_launch_by_launch(eng, crops, f"x1.0 shared batch {S} x {n}")
    print(f"\n[multistream osnet ops] {S} x {n} crops: {time.time() - t0:.1f} s; " +
          ", ".join(f"{k} {v:.3f}" for k, v in sorted(worst.items())))
