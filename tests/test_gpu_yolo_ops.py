"""Every launch of the detector engine, one at a time, against the float64 reference of what it computes
(oracle/nets64.py) at the input sizes the product runs; then the fp16 channels-last head decode and the DIoU-NMS on
the engine's own heads, and the NMS kernels at the edges of their blocks.

For each recorded launch (YoloEngine.trace describes it) the launch-by-launch test
  1. checks that every view it reads was written and still holds, bit for bit, what its producer wrote,
  2. snapshots every tensor it writes, runs it alone on the stream the replay uses, and checks that every element
     outside the declared output view (the other slices of a shared route buffer) is bit-identical,
  3. compares every output element with the float64 reference computed from the inputs as the kernel read them
     (teacher forcing), within the per-element bound of the kernel's rounding model.
A failure names the launch, the Darknet layers, the kind, the conv path, y / x / channel, got / want / bound and
error / bound.  With -s the largest error / bound per (kind, path) is printed.

The engines are built from synthetic BN-calibrated weights whose head objectness bias and gain keep the candidate
count of the scene frame between 100 and key_cap / 2 (a realistic decode / NMS load)."""
import ctypes as C
import time

import numpy as np
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

BUDGET = 1 << 30       # bytes of float64 working set per reference chunk (output rows per chunk follow from it)

# model -> synthetic head objectness bias and head gain (on the scene frame: about 490 / 1270 / 1450 / 2990 / 1370
# candidates pass conf_thresh), the (kind, conv path) pairs its launches reach
CASES = {
    'YOLOv4Tiny': (-1.0, 1.0, {('conv', 'tc'), ('conv', 'tma'), ('maxpool', None), ('upsample', None),
                               ('copy', None)}),
    'YOLOv4CSP': (-5.0, 0.25, {('conv', 'tc'), ('conv', 'tma'), ('conv+shortcut', 'tc'), ('conv+shortcut', 'tma'),
                               ('maxpool', None), ('upsample', None)}),
    'YOLOv4P5': (-5.0, 0.015, {('conv', 'tc'), ('conv', 'tma'), ('conv+shortcut', 'tc'),
                               ('conv+shortcut', 'tma'), ('maxpool', None), ('upsample', None)}),
    'YOLOv4P5_1280': (-5.0, 0.015, {('conv', 'tc'), ('conv', 'tma'), ('conv+shortcut', 'tc'),
                                    ('conv+shortcut', 'tma'), ('maxpool', None), ('upsample', None)}),
    'YOLOv4': (-5.0, 0.06, {('conv', 'tc'), ('conv', 'tma'), ('conv+shortcut', 'tc'), ('conv+shortcut', 'tma'),
                           ('maxpool', None), ('upsample', None)}),
}


def _bits(t):
    t = t.contiguous()
    return t.view(torch.int16) if t.dtype == torch.float16 else t.view(torch.int32)


def _region(v, t):
    """View v's elements in tensor t (a buffer of v's shape: [h][w][c_stride] fp16) as (1, h, w, c)."""
    return t.reshape(v.h, v.w, v.c_stride)[None, ..., v.c_off:v.c_off + v.c]


def _first_diff(a, b):
    """(y, x, channel) of the first element where a and b (1, h, w, c) differ in their bits."""
    i = int((_bits(a) != _bits(b)).reshape(-1).nonzero()[0])
    return tuple(int(v) for v in np.unravel_index(i, a.shape[1:]))


class Case:
    """One model: the engine with its synthetic weights, the detector around it, the scene frame through the
    detector's pre-processing and the engine's heads of that frame."""

    def __init__(self, name):
        from fastmot_b200 import models
        from fastmot_b200.detector import YOLODetector
        from fastmot_b200.engine import YoloEngine
        from fastmot_b200.models import darknet
        from fastmot_b200.synth import SyntheticScene
        bias, gain, self.expect = CASES[name]
        self.name = name
        m = self.model = models.YOLO.get_model(name)
        layers = darknet.BUILDERS[m.CFG](num_classes=m.NUM_CLASSES, anchors_per_head=len(m.ANCHORS[0]) // 2)
        weights = darknet.synthetic_weights(layers, 3, head_obj_bias=bias, num_classes=m.NUM_CLASSES, head_gain=gain)
        self.eng = YoloEngine(layers, m.INPUT_SHAPE[1:], weights, use_graph=False)
        self.det = YOLODetector((1920, 1080), tuple(range(m.NUM_CLASSES)), name, engine=self.eng)
        frame = SyntheticScene(200, seed=3).frame(0)
        self.det.preprocess(torch.as_tensor(frame).cuda())
        self.eng.forward(self.det.inp)
        torch.cuda.synchronize()

    def close(self):
        self.eng = self.det = None
        torch.cuda.empty_cache()


@pytest.fixture(scope="module", params=list(CASES))
def case(request):
    c = Case(request.param)
    yield c
    c.close()


# ------------------------------------------------------------------------------------------------ launch by launch
def _check(where, got, want, bound, r0=0):
    """Fails with the worst element of got (1, h, w, c; rows from r0) unless |got - want| <= bound everywhere."""
    from oracle import nets64 as R
    idx, r = R.worst(got, want, bound)
    if r > 1.0:
        pytest.fail(f"{where} at y/x/ch {(r0 + idx[1],) + idx[2:]}: got {float(got[idx]):.6g}, want "
                    f"{float(want[idx]):.6g}, bound {float(bound[idx]):.3g}, error/bound {r:.3g}")
    return r


def _conv_ref(eng, e, ins, got, where):
    """Conv (+ the fused shortcut) in chunks of output rows; returns the worst error / bound."""
    from oracle import nets64 as R
    i = e.ops[0]
    l = eng.layers[i]
    w, b = (a.double() for a in eng.params[i])
    k, s = l['size'], l.get('stride', 1)
    p = k // 2 if l.get('pad', 0) else 0
    act = l.get('activation', 'linear')
    x = ins[0]
    _, h, wi, cin = x.shape
    _, ho, wo, cout = got.shape
    rows = max(1, BUDGET // (8 * (wo * (cin * k * k + 12 * cout) + 2 * s * (wi + 2 * p) * cin)))
    ratio = 0.0
    for r0 in range(0, ho, rows):
        r1 = min(ho, r0 + rows)
        lo, hi = r0 * s - p, (r1 - 1) * s - p + k            # input rows of output rows r0 .. r1 - 1
        xs = F.pad(x[:, max(lo, 0):min(hi, h)].double(), (0, 0, p, p, max(0, -lo), max(0, hi - h)))
        res = ins[1][:, r0:r1] if e.kind == 'conv+shortcut' else None
        want, bound = R.conv(xs, w, b, s, 0, act, res=res, res_first=False)
        ratio = max(ratio, _check(where, got[:, r0:r1].double(), want, bound, r0))
    return ratio


def _reference_ratio(eng, e, ins, got, where):
    from oracle import nets64 as R
    if e.kind in ('conv', 'conv+shortcut'):
        return _conv_ref(eng, e, ins, got, where)
    if e.kind == 'maxpool':
        info = e.info
        if info['launch_src'] != info['src']:              # SPP: k x k over the k0 x k0 pool is the k + k0 - 1 window
            assert info['launch_size'] + eng.layers[info['launch_src']]['size'] - 1 == info['size'], (where, info)
        want, bound = R.maxpool(ins[0], info['size'], info['stride'])      # the declared window on the declared source
    elif e.kind == 'upsample':
        want, bound = R.upsample(ins[0], e.info['stride'])
    elif e.kind == 'copy':
        want, bound = R.copy(ins[0])
    elif e.kind == 'shortcut':
        want, bound = R.add_act(ins[0], ins[1], eng.layers[e.ops[0]].get('activation', 'linear'))
    else:
        raise NotImplementedError(e.kind)
    return _check(where, got.double(), want, bound)


def run_launch_by_launch(eng, label):
    """Runs eng's launches one by one on the input it holds and checks them; returns {(kind, path): worst ratio}."""
    from fastmot_b200.devmem import stream_ptr
    assert len(eng.trace) == len(eng.launches)
    last = {}                                               # buffer -> last launch that reads or writes it
    for k, e in enumerate(eng.trace):
        for v in e.ins + e.outs:
            last[v.t.data_ptr()] = k
    shadow = {eng.inp.data_ptr(): eng.inp.clone()}          # buffer -> what the launches so far left in it
    written = {eng.inp.data_ptr(): torch.ones(eng.inp.shape[-1], dtype=torch.bool)}
    worst = {}
    sp = stream_ptr()
    torch.cuda.synchronize()
    for k, e in enumerate(eng.trace):
        path = e.info.get('path')
        where = f"{label}: launch {k} ({e.kind}{'/' + path if path else ''}, layers {list(e.ops)})"
        ins = []
        for v in e.ins:                                     # 1. the inputs are what their producers wrote
            p = v.t.data_ptr()
            assert p in written and bool(written[p][v.c_off:v.c_off + v.c].all()), \
                (where, f"input '{v.name}' (channels {v.c_off}..{v.c_off + v.c}) read before it was written")
            was = _region(v, shadow[p])
            now = _region(v, v.t)
            if not torch.equal(_bits(now), _bits(was)):
                pytest.fail(f"{where}: input '{v.name}' was overwritten after its producer wrote it, first at "
                            f"y/x/ch {_first_diff(now, was)}")
            ins.append(was)
        before = {v.t.data_ptr(): v.t.clone() for v in e.outs}
        eng.launches[k](sp)                                 # 2. the launch alone
        torch.cuda.synchronize()
        for v in e.outs:
            p = v.t.data_ptr()
            after = v.t.clone()
            a, b = after.reshape(-1, v.c_stride), before[p].reshape(-1, v.c_stride)
            for sl in (slice(0, v.c_off), slice(v.c_off + v.c, v.c_stride)):
                if not torch.equal(_bits(a[:, sl]), _bits(b[:, sl])):
                    d = (_bits(a[:, sl]) != _bits(b[:, sl])).nonzero()[0]
                    pix, ch = int(d[0]), int(d[1]) + sl.start
                    pytest.fail(f"{where}: wrote outside its view '{v.name}' (channels {v.c_off}..{v.c_off + v.c} "
                                f"of {v.c_stride}) at y/x/ch {(pix // v.w, pix % v.w, ch)}")
            shadow[p] = after
            written.setdefault(p, torch.zeros(v.c_stride, dtype=torch.bool))[v.c_off:v.c_off + v.c] = True
        o = e.outs[0]                                       # 3. values
        got = _region(o, shadow[o.t.data_ptr()])
        r = _reference_ratio(eng, e, ins, got, f"{where}: output '{o.name}'")
        worst[(e.kind, path)] = max(worst.get((e.kind, path), 0.0), r)
        for p in [p for p, j in last.items() if j == k]:
            shadow.pop(p, None)
    return worst


def _report(label, eng, worst, t0):
    print(f"\n[yolo ops] {label} {eng.inp.shape[1]}x{eng.inp.shape[0]}: {len(eng.trace)} launches, "
          f"{time.time() - t0:.1f} s; max error/bound per (kind, path): " +
          ", ".join(f"{k}{'/' + p if p else ''} {v:.3f}" for (k, p), v in sorted(worst.items(), key=str)))


def test_yolo_engine_launch_by_launch(case):
    t0 = time.time()
    eng = case.eng
    reached = {(e.kind, e.info.get('path')) for e in eng.trace}
    assert reached == case.expect, reached
    _report(case.name, eng, run_launch_by_launch(eng, case.name), t0)


def test_yolo_engine_conv_tc_only_launch_by_launch(monkeypatch):
    """YOLOv4-csp 640 with every conv through conv_tc.cu (FM_CONV_TMA=0): its deep 40 x 40 / 20 x 20 layers and the
    heads are too few tiles to fill the GPU and split K, so both split-K reduces (8-channel and scalar) run."""
    monkeypatch.setenv("FM_CONV_TMA", "0")
    t0 = time.time()
    c = Case('YOLOv4CSP')
    try:
        assert {e.info.get('path') for e in c.eng.trace} == {'tc', None}
        _report("YOLOv4CSP, conv_tc only,", c.eng, run_launch_by_launch(c.eng, "YOLOv4CSP conv_tc only"), t0)
    finally:
        c.close()


# ------------------------------------------------------------------------------------------------ decode
def _decoded(det, heads):
    """decode64 of every head (NHWC [H][W][(5 + C) A] as the engine stores them), concatenated in candidate order."""
    from oracle import nets64 as R
    m = det.model
    wants, bounds = [], []
    for t, anchors, scale in zip(heads, m.ANCHORS, m.SCALES):
        want, bound = R.decode64(t.permute(2, 0, 1), anchors, scale, det.input_wh, m.NUM_CLASSES, m.NEW_COORDS,
                                 det.upscaled_sz, det.bbox_offset)
        wants.append(want)
        bounds.append(bound)
    return torch.cat(wants).cpu(), torch.cat(bounds).cpu()


def _keys(keys_dev, n):
    k = keys_dev[:n].cpu().numpy().view(np.uint64)
    return (k & np.uint64(0xffffff)).astype(np.int64), (k >> np.uint64(56)).astype(np.int64), \
        ((k >> np.uint64(24)) & np.uint64(0xffffffff)).astype(np.uint32)


def test_decode_of_engine_heads(case):
    """The product path (postprocess_heads_async on the engine's fp16 NHWC heads): the candidate set and the dense
    rows of decode64 on the same values; bit-exact for new-coords heads, within the __expf bound otherwise (a
    candidate whose score lies within its bound of conf_thresh may fall on either side)."""
    det, m = case.det, case.model
    det.postprocess_heads_async(case.eng.heads)
    det.postprocess()
    n = int(det._counter.item())
    assert 100 <= n <= det.key_cap // 2, n
    gidx, cls, sb = _keys(det._keys, n)
    dense = det._dense.cpu()
    want, bound = _decoded(det, case.eng.heads)
    lm = torch.as_tensor(det.label_mask)
    passing = lm[want[:, 5].long()] & (want[:, 7] >= det.conf_thresh)
    got_set, want_set = set(gidx.tolist()), set(passing.nonzero()[:, 0].tolist())
    assert len(got_set) == n
    if m.NEW_COORDS:
        assert got_set == want_set, (len(got_set - want_set), len(want_set - got_set))
    else:
        near = ((want[:, 7] - det.conf_thresh).abs() <= bound[:, 7]).nonzero()[:, 0].tolist()
        assert got_set ^ want_set <= set(near), sorted(got_set ^ want_set - set(near))[:10]
    rows = dense[gidx, :7].double()
    w, b = want[gidx, :7], bound[gidx, :7]
    err = (rows - w).abs()
    if m.NEW_COORDS:
        bad = (err > 0).any(1)
    else:
        bad = (err > b).any(1)
    if bool(bad.any()):
        j = int(bad.nonzero()[0])
        pytest.fail(f"{case.name}: candidate {gidx[j]}: dense row {rows[j].tolist()}, want {w[j].tolist()}, "
                    f"bound {b[j].tolist()}")
    assert np.array_equal(cls, dense[gidx, 5].numpy().astype(np.int64))
    assert np.array_equal(sb, ~dense[gidx, 4].numpy().view(np.uint32))


def test_nms_of_engine_candidates_teacher_forced(case):
    """oracle.detect.filter_dets on the kernel's own dense rows of the kept candidates equals the detector's output
    bit for bit (tlbr, label, conf)."""
    from oracle import detect
    det = case.det
    det.postprocess_heads_async(case.eng.heads)
    got = det.postprocess()
    n = int(det._counter.item())
    gidx = np.sort(_keys(det._keys, n)[0])                   # candidate order: the tie order of the sort keys
    rows = det._dense.cpu().numpy()[gidx, :7]
    want = detect.filter_dets(rows, (1.0, 1.0), (0.0, 0.0), det.label_mask, det.conf_thresh, det.nms_thresh,
                              det.max_area, det.min_aspect_ratio)
    assert len(got) == len(want[0]) > 0, (len(got), len(want[0]))
    assert np.array_equal(got.tlbr, want[0])
    assert np.array_equal(got.label, want[1])
    assert np.array_equal(got.conf, want[2])


def _decode(head, nhwc, shape, new_coords, anchors, scale, size=(1920.0, 1080.0), offset=(0.0, 140.0)):
    """fm_yolo_decode_filter on one head; returns (candidate indices ascending, their dense rows (n, 8))."""
    from fastmot_b200 import _lib
    from fastmot_b200.devmem import ptr, stream_ptr
    lib = _lib.load()
    A, nc, H, W = shape
    hd = _lib.FmYoloHead()
    for i, a in enumerate(anchors):
        hd.anchors[i] = float(a)
    hd.scale_x_y = float(scale)
    mask = torch.ones(nc, dtype=torch.uint8, device="cuda")
    dense = torch.zeros(A * H * W, 8, dtype=torch.float32, device="cuda")
    keys = torch.zeros(A * H * W, dtype=torch.int64, device="cuda")
    counter = torch.zeros(1, dtype=torch.int32, device="cuda")
    rc = lib.fm_yolo_decode_filter(ptr(head), 1 if head.dtype == torch.float16 else 0, nhwc, W, H, A, C.byref(hd), nc,
                                   416, 416, new_coords, 0, ptr(mask), 0.25, float(size[0]), float(size[1]),
                                   float(offset[0]), float(offset[1]), ptr(dense), ptr(keys), ptr(counter),
                                   keys.numel(), stream_ptr())
    _lib.check(rc, "fm_yolo_decode_filter")
    torch.cuda.synchronize()
    gidx = np.sort(_keys(keys, int(counter.item()))[0])
    return gidx, dense.cpu().numpy()[gidx]


@pytest.mark.parametrize("new_coords", [0, 1])
def test_decode_input_forms_agree_and_first_class_maximum_wins(new_coords):
    """fp16 / fp32 x channels-last / planar heads with the same values give identical dense tables; exact fp16 ties
    between class logits go to the first maximum; the rows are decode64's (exact for new coords)."""
    from oracle import nets64 as R
    A, nc, H, W = 3, 3, 13, 17
    anchors, scale = [10, 14, 23, 27, 37, 58], 1.05 if not new_coords else 2.0
    g = torch.Generator().manual_seed(21 + new_coords)
    t = torch.randn(A, 5 + nc, H, W, generator=g)
    if new_coords:
        t = torch.sigmoid(t * 1.5)
    else:
        t[:, 4] += 1.5
        t[:, 5:] += 1.0
    cls = t[:, 5:]
    pick = torch.randint(0, 3, (A, H, W), generator=g)
    cls[:, 1] = torch.where(pick == 1, cls[:, 0], cls[:, 1])                     # classes 0 and 1 tie
    cls[:, 2] = torch.where(pick == 1, torch.minimum(cls[:, 0], cls[:, 2]), cls[:, 2])
    top = torch.maximum(cls[:, 0], cls[:, 1]) + 0.25
    cls[:, 1] = torch.where(pick == 2, top, cls[:, 1])                           # classes 1 and 2 tie above 0
    cls[:, 2] = torch.where(pick == 2, top, cls[:, 2])
    planar16 = t.reshape(A * (5 + nc), H, W).half().cuda().contiguous()
    forms = {'planar fp16': (planar16, 0), 'planar fp32': (planar16.float(), 0),
             'nhwc fp16': (planar16.permute(1, 2, 0).contiguous(), 1),
             'nhwc fp32': (planar16.permute(1, 2, 0).float().contiguous(), 1)}
    out = {k: _decode(h, nhwc, (A, nc, H, W), new_coords, anchors, scale) for k, (h, nhwc) in forms.items()}
    g0, d0 = out['planar fp16']
    assert len(g0) > 50
    for k, (gi, d) in out.items():
        assert np.array_equal(gi, g0), k
        assert np.array_equal(d[:, :7].view(np.uint32), d0[:, :7].view(np.uint32)), k
    lv = planar16.reshape(A, 5 + nc, H, W)[:, 5:].float().cpu().numpy()
    first = np.argmax(lv, 1).reshape(-1)                                         # numpy: first maximum
    assert (pick.reshape(-1)[g0] > 0).sum() > 10
    assert np.array_equal(d0[:, 5].astype(np.int64), first[g0])
    want, bound = R.decode64(planar16, anchors, scale, (416, 416), nc, new_coords, (1920.0, 1080.0), (0.0, 140.0))
    want, bound = want.cpu()[g0, :7], bound.cpu()[g0, :7]
    err = (torch.as_tensor(d0[:, :7]).double() - want).abs()
    assert bool((err <= bound).all()), float((err / bound.clamp_min(1e-300)).max())
    if new_coords:
        assert float(err.max()) == 0.0


# ------------------------------------------------------------------------------------------------ NMS edges
def _nms_table(n, seed):
    """n candidates in clusters of overlapping boxes (jitter 2 / 8 / 20 px), two classes (some boxes duplicated
    across them), box_prob from eight levels (exact ties), quarter-pixel coordinates (rint half-way cases).
    Returns dense rows (n, 8) fp32 in pixels and the sort keys in shuffled order."""
    rng = np.random.default_rng(seed)
    nclu = max(1, n // 6)
    cx = 100.0 + 160.0 * (np.arange(nclu) % 40)
    cy = 100.0 + 200.0 * (np.arange(nclu) // 40)
    c = rng.integers(0, nclu, n)
    jit = np.array([2.0, 8.0, 20.0])[c % 3]
    w = rng.uniform(30, 90, n)
    h = w * rng.uniform(0.6, 3.0, n)
    x = cx[c] + rng.normal(0, 1, n) * jit - w / 2
    y = cy[c] + rng.normal(0, 1, n) * jit - h / 2
    rows = np.zeros((n, 8), np.float32)
    rows[:, 0], rows[:, 1] = np.round(x * 4) / 4, np.round(y * 4) / 4
    rows[:, 2], rows[:, 3] = np.round(w * 4) / 4, np.round(h * 4) / 4
    rows[:, 4] = (0.3 + 0.0875 * rng.integers(0, 8, n)).astype(np.float32)
    rows[:, 5] = rng.integers(0, 2, n)
    rows[:, 6] = np.float32(1.0) - np.float32(0.125) * rng.integers(0, 2, n)
    dup = rng.random(n) < 0.1                                   # the same box in the other class
    src = rng.integers(0, n, n)
    rows[dup, :5] = rows[src[dup], :5]
    rows[dup, 5] = 1 - rows[src[dup], 5]
    idx = rng.permutation(n).astype(np.uint64)
    bits = (~rows[idx.astype(np.int64), 4].view(np.uint32)).astype(np.uint64)
    keys = (rows[idx.astype(np.int64), 5].astype(np.uint64) << np.uint64(56)) | (bits << np.uint64(24)) | idx
    return rows, keys


def _nms(rows, keys, max_out, thresh=0.5, max_area=12000.0, min_ar=0.8):
    from fastmot_b200 import _lib
    from fastmot_b200.devmem import ptr, stream_ptr
    lib = _lib.load()
    cap = 16384
    keys_d = torch.zeros(cap, dtype=torch.int64, device="cuda")
    keys_d[:len(keys)] = torch.as_tensor(keys.view(np.int64)).cuda()
    dense = torch.as_tensor(rows).cuda()
    counter = torch.tensor([len(keys)], dtype=torch.int32, device="cuda")
    mask = torch.zeros(int(lib.fm_nms_mask_bytes(cap)), dtype=torch.uint8, device="cuda")
    o_t = torch.zeros(max_out, 4, dtype=torch.float64, device="cuda")
    o_l = torch.zeros(max_out, dtype=torch.int64, device="cuda")
    o_c = torch.zeros(max_out, dtype=torch.float64, device="cuda")
    meta = torch.zeros(2, dtype=torch.int32, device="cuda")
    rc = lib.fm_diou_nms_filter(ptr(keys_d), ptr(dense), ptr(counter), cap, thresh, max_area, min_ar, ptr(mask),
                                max_out, ptr(o_t), ptr(o_l), ptr(o_c), C.c_void_p(meta.data_ptr()),
                                C.c_void_p(meta.data_ptr() + 4), stream_ptr())
    _lib.check(rc, "fm_diou_nms_filter")
    torch.cuda.synchronize()
    cnt, status = meta.cpu().tolist()
    return cnt, status, o_t.cpu().numpy()[:cnt], o_l.cpu().numpy()[:cnt], o_c.cpu().numpy()[:cnt]


@pytest.mark.parametrize("n", [1, 63, 64, 65, 127, 2049, 16383, 16384])
def test_nms_block_edges_vs_filter_dets(n):
    """Sort, mask and blocked scan around the 64-candidate blocks, the 32-word survivor chunks, the power-of-two
    padding of the sort and the key capacity: bit-exact against oracle.detect.filter_dets."""
    from oracle import detect
    rows, keys = _nms_table(n, seed=n)
    cnt, status, tlbr, label, conf = _nms(rows, keys, max_out=16384)
    want = detect.filter_dets(rows[:, :7], (1.0, 1.0), (0.0, 0.0), np.ones(2, bool), 0.0, 0.5, 12000.0, 0.8)
    assert status == 0
    assert cnt == len(want[0]), (cnt, len(want[0]))
    assert np.array_equal(tlbr, want[0])
    assert np.array_equal(label, want[1])
    assert np.array_equal(conf, want[2])
    if n >= 2049:                                   # the table exercises suppression, both filters and both classes
        assert n // 8 < cnt < n * 3 // 4 and set(label.tolist()) == {0, 1}


def test_nms_more_survivors_than_max_out_is_status_2():
    """More survivors than output rows: status 2 (the host raises) and the first max_out rows still in order."""
    from oracle import detect
    rows, keys = _nms_table(2049, seed=5)
    cnt, status, tlbr, label, conf = _nms(rows, keys, max_out=100)
    want = detect.filter_dets(rows[:, :7], (1.0, 1.0), (0.0, 0.0), np.ones(2, bool), 0.0, 0.5, 12000.0, 0.8)
    assert len(want[0]) > 100
    assert status == 2 and cnt == 100
    assert np.array_equal(tlbr, want[0][:100]) and np.array_equal(label, want[1][:100])
    assert np.array_equal(conf, want[2][:100])


