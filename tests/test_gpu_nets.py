"""GPU numerics: conv-stack kernels and engines vs the fp32 PyTorch-CPU oracle (oracle/nets.py) with identical
synthetic weights.  Tolerance: fp16 storage + fp32 accumulation -> 2e-2 relative to the tensor scale."""
import ctypes as C

import numpy as np
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu


def _rel(got, want):
    return float((got - want).abs().max() / (want.abs().max() + 1e-6))


CONV_CASES = [
    # n, h, w, cin, cout, k, stride, act, cin_stride, cin_off, cout_stride, cout_off, residual
    (1, 40, 40, 8, 32, 3, 2, 'leaky', 8, 0, 32, 0, False),
    (1, 33, 29, 64, 64, 3, 1, 'mish', 64, 0, 64, 0, False),
    (2, 16, 24, 32, 48, 1, 1, 'linear', 96, 32, 80, 16, False),
    (1, 20, 20, 128, 256, 3, 2, 'leaky', 128, 0, 256, 0, False),
    (3, 32, 16, 8, 16, 7, 2, 'relu', 8, 0, 16, 0, False),
    (1, 30, 30, 4, 16, 3, 1, 'relu', 4, 0, 16, 0, False),
    (1, 26, 26, 256, 18, 1, 1, 'logistic', 256, 0, 18, 0, False),
    (1, 24, 24, 64, 64, 3, 1, 'relu', 64, 0, 64, 0, True),
    (4, 64, 32, 16, 16, 1, 1, 'swish', 16, 0, 16, 0, False),
]


def _run_conv(fn_name, case, seed=0):
    """case: the CONV_CASES fields, optionally followed by res_first: FM_ACT_AFTER_RESIDUAL, act(conv + b + res)
    instead of the Darknet order act(conv + b) + res."""
    from fastmot_b200 import _lib
    from fastmot_b200.devmem import ptr, stream_ptr
    from fastmot_b200.engine import ACT_AFTER_RESIDUAL, _conv_desc
    from fastmot_b200.models.darknet import ACTS
    from oracle.nets import _act
    lib = _lib.load()
    ws = torch.empty(32 << 20, dtype=torch.uint8, device="cuda")   # enables split-K for small-M / large-K shapes
    n, h, w, cin, cout, k, stride, act, cis, cio, cos, coo, use_res = case[:13]
    res_first = len(case) > 13 and case[13]
    g = torch.Generator().manual_seed(seed)
    pad = k // 2
    ho, wo = (h + 2 * pad - k) // stride + 1, (w + 2 * pad - k) // stride + 1
    xin = (torch.randn(n, h, w, cis, generator=g) * 0.5).half()
    wt = (torch.randn(cout, k, k, cin, generator=g) * (2.0 / (k * k * cin)) ** 0.5).half()
    bias = torch.randn(cout, generator=g) * 0.1
    res = (torch.randn(n, ho, wo, cout, generator=g) * 0.5).half() if use_res else None
    out = torch.zeros(n, ho, wo, cos, dtype=torch.float16)
    d = _conv_desc(n, h, w, cin, cis, cio, ho, wo, cout, cos, coo, k, stride, pad,
                   ACTS[act] | (ACT_AFTER_RESIDUAL if res_first else 0), ws=ws)
    if use_res:
        d.res_stride, d.res_offset = cout, 0
    if fn_name == 'fm_conv2d_tc' and not lib.fm_conv2d_tc_supported(C.byref(d)):
        return None
    if fn_name == 'fm_conv2d_tma':
        assert lib.fm_conv2d_tma_supported(C.byref(d)), case
    xd, wd, bd, od = xin.cuda(), wt.cuda(), bias.cuda(), out.cuda()
    rd = res.cuda() if use_res else None
    rc = getattr(lib, fn_name)(C.byref(d), ptr(xd), ptr(wd), ptr(bd), ptr(rd), ptr(od), stream_ptr())
    _lib.check(rc, fn_name)
    torch.cuda.synchronize()
    got = od.cpu().float()
    xs = xin[..., cio:cio + cin].float().permute(0, 3, 1, 2)
    y = F.conv2d(xs, wt.float().permute(0, 3, 1, 2), bias, stride=stride, padding=pad)
    if res_first:
        y = _act(y + res.float().permute(0, 3, 1, 2), act)
    else:
        y = _act(y, act)
        if use_res:
            y = y + res.float().permute(0, 3, 1, 2)
    want = y.permute(0, 2, 3, 1)
    assert _rel(got[..., coo:coo + cout], want) < 4e-3, (fn_name, case, _rel(got[..., coo:coo + cout], want))
    untouched = torch.cat([got[..., :coo], got[..., coo + cout:]], -1)
    assert float(untouched.abs().max()) == 0.0 if untouched.numel() else True
    return True


# FM_ACT_AFTER_RESIDUAL (res_first, last field): out = act(conv + b + res), the order of OSNet's conv3 + add + ReLU
RES_FIRST_SIMT = [
    (1, 24, 24, 64, 64, 3, 1, 'leaky', 64, 0, 64, 0, True, True),
    (2, 16, 8, 40, 20, 1, 1, 'relu', 40, 0, 20, 0, True, True),
]


@pytest.mark.parametrize("case", CONV_CASES + RES_FIRST_SIMT)
def test_conv_simt_vs_torch(case):
    assert _run_conv('fm_conv2d_simt', case)


# every epilogue branch of conv_tc.cu with FM_ACT_AFTER_RESIDUAL (shapes chosen from fm_conv2d_tc / launch_tc)
RES_FIRST_TC = [
    (2, 16, 8, 96, 384, 1, 1, 'relu', 96, 0, 384, 0, True, True),      # nk 2, no split, 8-aligned: epilogue_staged
    (1, 12, 12, 64, 36, 1, 1, 'leaky', 64, 0, 48, 0, True, True),      # cout 36: epilogue_store32, 16-aligned stores
    (1, 12, 12, 64, 36, 1, 1, 'leaky', 64, 0, 40, 0, True, True),      # stride 40: epilogue_store32 element-wise
    (1, 10, 10, 512, 64, 3, 1, 'leaky', 512, 0, 64, 0, True, True),    # 1 tile, nk 72: split-K, 8-wide reduce
    (1, 10, 10, 640, 20, 1, 1, 'leaky', 640, 0, 20, 0, True, True),    # 1 tile, nk 10, cout 20: scalar reduce
]


@pytest.mark.parametrize("case", RES_FIRST_TC)
def test_conv_tc_act_after_residual(case):
    assert _run_conv('fm_conv2d_tc', case)


@pytest.mark.parametrize("case", CONV_CASES + [
    (1, 80, 80, 128, 128, 3, 1, 'mish', 128, 0, 128, 0, False),
    (1, 20, 20, 512, 1024, 3, 1, 'mish', 512, 0, 1024, 0, False),
    (8, 64, 32, 64, 64, 1, 1, 'relu', 64, 0, 64, 0, False),
    (1, 40, 40, 256, 512, 3, 2, 'leaky', 256, 0, 512, 0, False),
    (2, 16, 8, 96, 384, 1, 1, 'linear', 96, 0, 384, 0, True),
    (1, 13, 13, 512, 256, 1, 1, 'leaky', 1024, 512, 256, 0, False),
    (1, 20, 20, 1024, 512, 3, 1, 'mish', 1024, 0, 512, 0, True),      # split-K with residual
    (1, 40, 40, 256, 256, 3, 1, 'leaky', 256, 0, 512, 256, False),    # split-K into a concat slice
    (1, 10, 10, 640, 24, 1, 1, 'logistic', 640, 0, 24, 0, False),     # split-K, ragged cout
    (40, 64, 32, 64, 64, 1, 1, 'linear', 64, 0, 64, 0, False),        # persistent small-K variant (640 tiles)
    (40, 64, 32, 64, 256, 1, 1, 'relu', 64, 0, 256, 0, True),         # small-K, 2 N tiles, residual
    (40, 64, 32, 96, 96, 1, 1, 'relu', 96, 0, 96, 0, False),          # small-K with 2 K slices (K = 96)
    (40, 64, 32, 128, 24, 1, 1, 'linear', 128, 0, 24, 0, False),      # small-K, ragged cout, BN = 32
])
def test_conv_tc_vs_torch(case):
    r = _run_conv('fm_conv2d_tc', case)
    if r is None:
        pytest.skip("shape not handled by the wgmma path (falls back to the SIMT kernel)")


TMA_CASES = [
    # n, h, w, cin, cout, k, stride, act, cin_stride, cin_off, cout_stride, cout_off, residual
    (1, 80, 80, 128, 128, 3, 1, 'mish', 128, 0, 128, 0, False),       # 16x8 rectangles, cluster of 8 (18 K slices)
    (1, 80, 80, 128, 128, 3, 1, 'mish', 128, 0, 128, 0, True),        # fused CSP shortcut
    (1, 80, 80, 256, 128, 1, 1, 'mish', 256, 0, 256, 128, False),     # 1x1 into a concat slice, 2-way split
    (1, 80, 80, 128, 256, 3, 1, 'leaky', 128, 0, 256, 0, False),      # 100 tiles: no split
    (1, 40, 40, 256, 256, 3, 1, 'mish', 256, 0, 256, 0, True),        # 40x3 rectangles (120 rows used), split 8
    (1, 40, 40, 512, 256, 1, 1, 'mish', 512, 0, 256, 0, False),       # 64-wide filter tiles, split 4
    (1, 40, 40, 256, 512, 3, 1, 'leaky', 256, 0, 512, 0, False),
    (1, 20, 20, 512, 512, 3, 1, 'mish', 512, 0, 512, 0, False),       # 20x6 rectangles, 72 K slices
    (1, 20, 20, 1024, 512, 1, 1, 'mish', 2048, 1024, 512, 0, False),  # input channel slice of a concat buffer
    (1, 20, 20, 2048, 512, 1, 1, 'leaky', 2048, 0, 512, 0, False),    # SPP output: 32 K slices
    (1, 20, 20, 512, 1024, 3, 1, 'mish', 512, 0, 1024, 0, False),
    (1, 13, 13, 512, 256, 1, 1, 'leaky', 1024, 512, 256, 0, False),   # ragged last tile (169 pixels)
    (1, 19, 23, 64, 64, 3, 1, 'relu', 64, 0, 64, 0, True),            # odd plane, single K chunk per tap
    (1, 26, 26, 256, 40, 1, 1, 'logistic', 256, 0, 40, 0, False),     # cout < filter tile (rows beyond cout masked)
    (3, 16, 8, 192, 384, 1, 1, 'linear', 192, 0, 384, 0, True),       # batch > 1 (flattened 1x1), 3 K slices
    (40, 64, 32, 256, 256, 1, 1, 'relu', 256, 0, 256, 0, False),      # OSNet transition geometry: 640 tiles, no split
    (1, 160, 160, 64, 64, 3, 1, 'mish', 64, 0, 128, 64, False),       # 200 tiles, concat slice
    (1, 6, 5, 64, 32, 3, 1, 'linear', 64, 0, 32, 0, False),           # plane smaller than one tile
    (1, 80, 80, 128, 256, 3, 2, 'mish', 128, 0, 256, 0, False),       # stride 2 through the 5-D parity view
    (1, 40, 40, 256, 512, 3, 2, 'leaky', 256, 0, 512, 0, False),      # stride 2, 36 K slices, split
    (1, 320, 320, 64, 128, 3, 2, 'mish', 64, 0, 128, 0, False),       # stride 2, 200 tiles
    (1, 26, 22, 64, 64, 3, 2, 'relu', 128, 64, 64, 0, False),         # stride 2, channel slice in, ragged tiles
    (1, 40, 40, 512, 18, 1, 1, 'logistic', 512, 0, 18, 0, False),     # detection head: 18 channels, element-wise stores
    (1, 20, 20, 1024, 18, 1, 1, 'linear', 1024, 0, 18, 0, False),     # head with a deep K split
]


# conv_tma.cu epilogue with FM_ACT_AFTER_RESIDUAL; plans from fm_conv2d_tma / pick_split
RES_FIRST_TMA = [
    (4, 64, 32, 128, 128, 1, 1, 'leaky', 128, 0, 128, 0, True, True),  # 64-wide, 128 tiles, nk 2: S == 1, vector
    (1, 20, 20, 512, 256, 3, 1, 'leaky', 512, 0, 256, 0, True, True),  # 4 x 2 tiles, nk 72: S > 1, vector
    (1, 26, 26, 64, 36, 1, 1, 'leaky', 64, 0, 36, 0, True, True),      # cout 36, nk 1: S == 1, element-wise
    (1, 20, 20, 1024, 18, 1, 1, 'leaky', 1024, 0, 18, 0, True, True),  # cout 18, 4 tiles, nk 16: S > 1, element-wise
]


@pytest.mark.parametrize("case", TMA_CASES + RES_FIRST_TMA)
def test_conv_tma_vs_torch(case):
    """TMA-fed wgmma conv with in-cluster split-K (csrc/conv_tma.cu) vs fp32 torch."""
    assert _run_conv('fm_conv2d_tma', case)


@pytest.mark.parametrize("split", ["1", "2", "5", "8"])
def test_conv_tma_split_sizes_agree(split, monkeypatch):
    """Every cluster size gives the same layer (fp32 partial sums; order of summation differs -> tolerance)."""
    import subprocess, sys, os
    code = ("import sys; sys.path.insert(0, 'tests'); import test_gpu_nets as t; "
            "[t._run_conv('fm_conv2d_tma', c) for c in (t.TMA_CASES[4], t.TMA_CASES[7], t.TMA_CASES[9])]")
    env = dict(os.environ, FM_CONV_TMA_SPLIT=split)
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    r = subprocess.run([sys.executable, "-c", code], cwd=root, env=env, capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stderr[-2000:]


def _yolo_vs_oracle(name, hw, tol):
    from fastmot_b200.engine import YoloEngine
    from fastmot_b200.models import darknet
    from oracle import nets
    layers = darknet.BUILDERS[name]()
    weights = darknet.synthetic_weights(layers, 3, head_obj_bias=-3.0)
    eng = YoloEngine(layers, hw, weights, use_graph=False)
    g = torch.Generator().manual_seed(1)
    x = torch.rand(1, 3, hw[0], hw[1], generator=g)
    inp = torch.zeros(hw[0], hw[1], 8, dtype=torch.float16)
    inp[..., :3] = x[0].permute(1, 2, 0).half()
    heads = eng.forward(inp.cuda())
    torch.cuda.synchronize()
    want = nets.run_darknet(layers, weights, inp[..., :3].float().permute(2, 0, 1)[None], nets.fp16_roundtrip)
    assert len(heads) == len(want)
    for hg, hw_ in zip(heads, want):
        got = hg.cpu().float().permute(2, 0, 1)
        assert got.shape == hw_.shape
        assert _rel(got, hw_) < tol, (name, _rel(got, hw_))
    return eng


@pytest.mark.parametrize("shape", [
    (3, 64, 32, 64),     # OSNet stage 1 geometry: shared-memory tiled kernel, 8 full strips
    (2, 20, 12, 24),     # ragged last strip (20 = 2 * 8 + 4), 3 channel groups
    (2, 16, 8, 128),     # stage 3 geometry
    (1, 5, 8, 16),       # fewer rows than a strip: untiled vec4 kernel
    (1, 9, 7, 8),        # width not a multiple of 4: per-pixel kernel
])
def test_dwconv3_vs_torch(shape):
    """Depthwise 3x3 s1 p1 + bias + ReLU (OSNet Lite 3x3 second half) on every kernel variant."""
    from fastmot_b200 import _lib
    from fastmot_b200.devmem import ptr, stream_ptr
    lib = _lib.require_device()
    n, h, w, c = shape
    g = torch.Generator().manual_seed(11)
    x = torch.randn(n, h, w, c, generator=g).half()
    wt = (torch.randn(9, c, generator=g) * 0.3).half()
    b = torch.randn(c, generator=g) * 0.1
    xd, wd_, bd = x.cuda(), wt.cuda(), b.cuda()
    out = torch.empty(n, h, w, c, dtype=torch.float16, device="cuda")
    _lib.check(lib.fm_dwconv3(ptr(xd), ptr(wd_), ptr(bd), ptr(out), n, h, w, c, 5, stream_ptr()), "fm_dwconv3")
    torch.cuda.synchronize()
    ref = F.conv2d(x.float().permute(0, 3, 1, 2), wt.float().t().reshape(c, 1, 3, 3), b, padding=1, groups=c)
    ref = F.relu(ref).permute(0, 2, 3, 1)
    assert _rel(out.float().cpu(), ref) < 5e-3


def test_yolov4_tiny_engine_vs_oracle():
    eng = _yolo_vs_oracle('yolov4-tiny', (416, 416), 2e-2)
    assert eng.n_tc + eng.n_simt == 21


@pytest.mark.parametrize("name,hw", [("yolov4-csp", (256, 256)), ("yolov4-p5", (256, 256)), ("yolov4", (256, 256)),
                                     ("yolov4-csp", (640, 640))])      # the benchmarked detector shape
def test_deep_yolo_engine_layerwise(name, hw):
    """Deep random-weight nets amplify rounding noise end to end (no trained BN statistics), so every layer is
    checked against fp32 torch applied to the ENGINE's own input for that layer (teacher forcing): covers each
    conv + activation, shortcut, route/concat placement, group split, SPP max-pools and upsampling."""
    from fastmot_b200.engine import YoloEngine
    from fastmot_b200.models import darknet
    from oracle.nets import _act, _same_upper_pool
    layers = darknet.BUILDERS[name]()
    weights = darknet.synthetic_weights(layers, 3, head_obj_bias=-3.0)
    eng = YoloEngine(layers, hw, weights, use_graph=False)
    x = torch.rand(hw[0], hw[1], 8).half()
    x[..., 3:] = 0
    eng.forward(x.cuda())
    torch.cuda.synchronize()

    def fetch(i):
        t, c, cs, co, h, w = eng.views[i]
        return t.reshape(h, w, cs)[..., co:co + c].float().cpu().permute(2, 0, 1)[None]

    worst = 0.0
    for i, l in enumerate(eng.layers):
        t = l['type']
        src = fetch(i - 1) if i else x[..., :3].float().permute(2, 0, 1)[None]
        if t == 'convolutional':
            w, b = weights[i]
            k = l['size']
            want = _act(F.conv2d(src, torch.as_tensor(w).half().float().permute(0, 3, 1, 2), torch.as_tensor(b),
                                 stride=l.get('stride', 1), padding=k // 2), l.get('activation', 'linear'))
            if i + 1 in eng.fused_shortcuts:      # the shortcut's add runs in this conv's epilogue
                want = want + fetch(eng.layers[i + 1]['from_abs'])
        elif t == 'shortcut' and i in eng.fused_shortcuts:
            assert eng.views[i][0].data_ptr() == eng.views[i - 1][0].data_ptr()
            continue
        elif t == 'maxpool':
            want = _same_upper_pool(src, l['size'], l['stride'])
        elif t == 'upsample':
            want = F.interpolate(src, scale_factor=2, mode='nearest')
        elif t == 'shortcut':
            want = src + fetch(l['from_abs'])
        elif t == 'route':
            g, gid = l.get('groups', 1), l.get('group_id', 0)
            parts = []
            for s_ in l['layers_abs']:
                o = fetch(s_)
                c = o.shape[1] // g
                parts.append(o[:, gid * c:(gid + 1) * c])
            want = torch.cat(parts, 1)
        else:
            continue
        got = fetch(i)
        assert got.shape == want.shape, (i, t)
        r = _rel(got, want)
        worst = max(worst, r)
        assert r < 6e-3, (name, i, t, r)
    assert len(eng.heads) == 3


def test_yolo_engine_graph_replay_matches_eager():
    from fastmot_b200.engine import YoloEngine
    from fastmot_b200.models import darknet
    layers = darknet.yolov4_tiny()
    weights = darknet.synthetic_weights(layers, 3)
    a = YoloEngine(layers, (416, 416), weights, use_graph=False)
    b = YoloEngine(layers, (416, 416), weights, use_graph=True)
    x = torch.rand(416, 416, 8, device="cuda").half()
    ha = [h.clone() for h in a.forward(x)]
    for _ in range(3):
        hb = b.forward(x)
    torch.cuda.synchronize()
    for p, q in zip(ha, hb):
        assert torch.equal(p, q)


@pytest.mark.parametrize("width", [0.25, 1.0])
def test_osnet_engine_vs_oracle(width):
    from fastmot_b200.engine import OSNetEngine
    from oracle import nets
    eng = OSNetEngine(width, max_batch=6, use_graph=False)
    g = torch.Generator().manual_seed(2)
    x = torch.randn(6, 3, 256, 128, generator=g)
    inp = torch.zeros(6, 256, 128, 8, dtype=torch.float16)
    inp[..., :3] = x.permute(0, 2, 3, 1).half()
    eng.load_nhwc8(inp.cuda())
    got = eng.forward().cpu()
    want = nets.run_osnet(eng.ops, eng.weights, inp[..., :3].float().permute(0, 3, 1, 2), nets.fp16_roundtrip)
    assert got.shape == want.shape == (6, 512)
    np.testing.assert_allclose(got.norm(dim=1).numpy(), 1.0, atol=1e-4)
    assert float((got - want).abs().max()) < 5e-3, float((got - want).abs().max())


def test_feature_extractor_end_to_end():
    from fastmot_b200 import FeatureExtractor
    from fastmot_b200.synth import SyntheticScene
    from oracle import nets, detect
    sc = SyntheticScene(20, seed=8)
    frame = sc.frame(0)
    tl = sc.detections(0)[0]
    fe = FeatureExtractor('OSNet025', use_graph=False)
    emb = np.asarray(fe(frame, tl))
    assert emb.shape == (20, 512)
    crops = torch.as_tensor(detect.roi_preprocess_fixedpoint(frame, tl))
    eng = fe._engine(20)
    want = nets.run_osnet(eng.ops, eng.weights, crops.half().float(), nets.fp16_roundtrip).numpy()
    assert np.abs(emb - want).max() < 5e-3
    assert fe.metric == 'euclidean'
    assert len(np.asarray(fe(frame, np.zeros((0, 4))))) == 0


def test_yolo_detector_end_to_end_vs_oracle_pipeline():
    from fastmot_b200 import YOLODetector, models
    from fastmot_b200.synth import SyntheticScene
    from oracle import nets, detect
    frame = SyntheticScene(30, seed=2).frame(0)
    det = YOLODetector((1920, 1080), (0,), 'YOLOv4Tiny', min_aspect_ratio=0.2)
    got = det(frame)
    model = models.YOLO.get_model('YOLOv4Tiny')
    roi, up, off = detect.letterbox_geometry((1920, 1080), (416, 416), model.LETTERBOX)
    x = torch.as_tensor(detect.letterbox(frame, (416, 416), roi)).half().float()[None]
    eng = det.backend
    weights = {i: (eng.params[i][0].float().cpu().numpy()[..., :3] if i == 0 else eng.params[i][0].float().cpu().numpy(),
                   eng.params[i][1].cpu().numpy()) for i in eng.params}
    heads = nets.run_darknet(eng.layers, weights, x, nets.fp16_roundtrip)
    dec = [detect.yolo_decode(h.numpy(), a, s, (416, 416), 1, False)
           for h, a, s in zip(heads, model.ANCHORS, model.SCALES)]
    want = detect.filter_dets(np.concatenate(dec), up, off, det.label_mask, 0.25, 0.5, 800000, 0.2)
    # fp16 conv noise moves scores across the threshold for a few candidates: compare as sets with tolerance
    assert abs(len(got) - len(want[0])) <= max(3, len(want[0]) // 10), (len(got), len(want[0]))
    if len(want[0]) and len(got):
        d = np.abs(got.tlbr[:, None, :] - want[0][None, :, :]).max(-1)
        assert (d.min(1) <= 2).mean() > 0.8


def test_darknet_cfg_and_weights_files_through_the_gpu_engine(tmp_path):
    """SURVEY.md 8(f1): a Darknet .cfg + .weights pair on disk (written from the synthetic YOLOv4-tiny weights) goes
    through parse_cfg / load_weights into YoloEngine and must give the heads of the engine built directly from the
    builder's layer list and weights (the only difference is one fp32 rounding of the identity BN scale)."""
    from fastmot_b200.engine import YoloEngine
    from fastmot_b200.models import darknet
    layers = darknet.yolov4_tiny()
    weights = darknet.synthetic_weights(layers, 3)
    cfg_path, w_path = tmp_path / "net.cfg", tmp_path / "net.weights"
    cfg_path.write_text(darknet.to_cfg(layers, 416, 416))
    darknet.save_weights(str(w_path), layers, weights, 3)
    net, layers2 = darknet.parse_cfg(cfg_path.read_text())
    assert (net['width'], net['height']) == (416, 416) and len(layers2) == len(layers)
    loaded = darknet.load_weights(str(w_path), layers2, 3)
    assert sorted(loaded) == sorted(weights)
    for i in weights:
        np.testing.assert_allclose(loaded[i][0], weights[i][0], rtol=3e-7, atol=1e-9)
        np.testing.assert_array_equal(loaded[i][1], np.asarray(weights[i][1], np.float32))
    a = YoloEngine(layers, (416, 416), weights, use_graph=False)
    b = YoloEngine(layers2, (416, 416), loaded, use_graph=False)
    x = torch.rand(416, 416, 8, device="cuda").half()
    x[..., 3:] = 0
    ha = [h.clone().float() for h in a.forward(x)]
    hb = [h.float() for h in b.forward(x)]
    assert len(ha) == len(hb) == 2
    for p, q in zip(ha, hb):
        assert p.shape == q.shape
        assert float((p - q).abs().max()) <= 2e-3 * float(p.abs().max() + 1)
