"""CPU checks of the seven YOLO models added to the four the detector first ran (YOLOv3, YOLOv3-SPP, YOLOv3-tiny,
YOLOv4x-mish, YOLOv4-csp-swish, YOLOv4-csp-x-swish, YOLOv4-P6): their builders, their descriptors against the
reference's registry, the head-table validation, the Darknet file round trip and the float64 executor."""
import os
import re

import numpy as np
import pytest
import torch

from fastmot_b200 import models
from fastmot_b200.models import darknet
from fastmot_b200.models.yolo import MAX_ANCHORS, check_heads

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

NEW = ['YOLOv3', 'YOLOv3SPP', 'YOLOv3Tiny', 'YOLOv4xMish', 'YOLOv4CSPSwish', 'YOLOv4CSPxSwish', 'YOLOv4P6']
ALL = ['YOLOv4', 'YOLOv4CSP', 'YOLOv4P5', 'YOLOv4Tiny'] + NEW

# fastmot/models/yolo.py of the reference, restated: name -> (line, NUM_CLASSES, LETTERBOX, NEW_COORDS, INPUT_SHAPE,
# LAYER_FACTORS, SCALES, ANCHORS)
_CSP_ANCHORS = [[12, 16, 19, 36, 40, 28], [36, 75, 76, 55, 72, 146], [142, 110, 192, 243, 459, 401]]
_V3_ANCHORS = [[116, 90, 156, 198, 373, 326], [30, 61, 62, 45, 59, 119], [10, 13, 16, 30, 33, 23]]
REFERENCE = {
    'YOLOv4xMish': (185, 1, True, True, (3, 640, 640), [8, 16, 32], [2.0, 2.0, 2.0], _CSP_ANCHORS),
    'YOLOv4CSPSwish': (199, 1, True, True, (3, 640, 640), [8, 16, 32], [2.0, 2.0, 2.0], _CSP_ANCHORS),
    'YOLOv4CSPxSwish': (213, 1, True, True, (3, 640, 640), [8, 16, 32], [2.0, 2.0, 2.0], _CSP_ANCHORS),
    'YOLOv4P6': (241, 1, True, True, (3, 1280, 1280), [8, 16, 32, 64], [2.0, 2.0, 2.0, 2.0],
                 [[13, 17, 31, 25, 24, 51, 61, 45], [61, 45, 48, 102, 119, 96, 97, 189],
                  [97, 189, 217, 184, 171, 384, 324, 451], [324, 451, 545, 357, 616, 618, 1024, 1024]]),
    'YOLOv3': (267, 1, False, False, (3, 416, 416), [32, 16, 8], [1.0, 1.0], _V3_ANCHORS),
    'YOLOv3SPP': (279, 1, False, False, (3, 608, 608), [32, 16, 8], [1.0, 1.0], _V3_ANCHORS),
    'YOLOv3Tiny': (291, 1, False, False, (3, 416, 416), [32, 16], [1.0, 1.0],
                   [[81, 82, 135, 169, 344, 319], [10, 14, 23, 27, 37, 58]]),
}


def _layers(m, num_classes=None):
    return darknet.BUILDERS[m.CFG](num_classes=m.NUM_CLASSES if num_classes is None else num_classes,
                                   anchors_per_head=len(m.ANCHORS[0]) // 2)


# ------------------------------------------------------------------------------------------------ builders
def test_published_flops_of_the_v3_builders():
    """pjreddie/darknet's published figures at 80 classes: YOLOv3-416 65.86, YOLOv3-tiny 5.56 and YOLOv3-SPP-608
    141.45 BFLOPs."""
    for cfg, hw, want in (('yolov3', 416, 65.86), ('yolov3-tiny', 416, 5.56), ('yolov3-spp', 608, 141.45)):
        got = darknet.count_flops(darknet.BUILDERS[cfg](num_classes=80), 3, hw, hw) / 1e9
        assert abs(got - want) < 0.01, (cfg, got)


def test_v3_builders_have_the_layer_counts_of_the_published_cfgs():
    """yolov3.cfg: 107 layers (75 convs, the routes at 83 / 86 / 95 / 98 reading 79, 61, 91 and 36); yolov3-spp.cfg:
    114; yolov3-tiny.cfg: 24, its sixth max-pool 2 x 2 at stride 1."""
    v3 = darknet.yolov3()
    assert len(v3) == 107 and sum(l['type'] == 'convolutional' for l in v3) == 75
    assert [(i, l['layers']) for i, l in enumerate(v3) if l['type'] == 'route'] == \
        [(83, [79]), (86, [-1, 61]), (95, [91]), (98, [-1, 36])]
    assert [i for i, l in enumerate(v3) if l['type'] == 'yolo'] == [82, 94, 106]
    spp = darknet.yolov3_spp()
    assert len(spp) == 114 and [i for i, l in enumerate(spp) if l['type'] == 'yolo'] == [89, 101, 113]
    assert [(l['size'], l['stride']) for l in spp if l['type'] == 'maxpool'] == [(5, 1), (9, 1), (13, 1)]
    tiny = darknet.yolov3_tiny()
    assert len(tiny) == 24 and [i for i, l in enumerate(tiny) if l['type'] == 'yolo'] == [16, 23]
    assert [(l['size'], l['stride']) for l in tiny if l['type'] == 'maxpool'] == [(2, 2)] * 5 + [(2, 1)]


def test_scaled_yolov4_builders_counts_and_scaling():
    """The published Darknet cfgs of the Scaled-YOLOv4 models are not part of the reference, so these counts pin this
    restatement (ScaledYOLOv4 models/yolov4-csp-x.yaml and yolov4-p6.yaml) rather than a file: layers, convs and
    BFLOPs at 80 classes.  The x models are yolov4-csp at width x 1.25 (every conv) and depth x 1.33."""
    def counts(cfg, hw, **kw):
        layers = darknet.BUILDERS[cfg](num_classes=80, **kw)
        return (len(layers), sum(l['type'] == 'convolutional' for l in layers),
                round(darknet.count_flops(layers, 3, hw, hw) / 1e9, 2))
    assert counts('yolov4-csp', 640) == counts('yolov4-csp-swish', 640) == (177, 117, 123.18)
    assert counts('yolov4x-mish', 640) == counts('yolov4-csp-x-swish', 640) == (211, 143, 234.38)
    assert counts('yolov4-p6', 1280, anchors_per_head=4) == (302, 205, 726.46)
    csp, x = darknet.yolov4_csp(80), darknet.yolov4_csp_x(80)
    widths = lambda ls: [l['filters'] for l in ls if l['type'] == 'convolutional' and l['activation'] == 'mish']
    assert {w * 5 // 4 for w in widths(csp)} == set(widths(x)) == {40, 80, 160, 320, 640, 1280}
    units = lambda ls: sum(l['type'] == 'shortcut' for l in ls)
    assert (units(csp), units(x)) == (1 + 2 + 8 + 8 + 4, 1 + 3 + 11 + 11 + 5)
    acts = {l['activation'] for l in darknet.BUILDERS['yolov4-csp-x-swish']() if l['type'] == 'convolutional'}
    assert acts == {'swish', 'logistic'}
    # P6: a sixth stage at stride 64 (20 x 20 at 1280) with the SPP block on it, four heads
    p6 = darknet.yolov4_p6()
    res, shapes = darknet.infer_shapes(p6, 3, 1280, 1280)
    assert max(shapes[i][0] for i, l in enumerate(res) if l['type'] == 'convolutional' and shapes[i][1] == 20) == 1024
    assert [shapes[i][1:] for i, l in enumerate(res) if l['type'] == 'maxpool'] == [(20, 20)] * 3


def _scaled_yolov4_three_levels(depths, widths, neck_n, num_classes, anchors_per_head, act='mish'):
    """The three-level Scaled-YOLOv4 builder the csp and p5 models were built with before it took any number of
    levels, kept verbatim so the generalised one is held to the same layer lists."""
    b = darknet._B()
    out_c = anchors_per_head * (5 + num_classes)
    b.conv(32, 3, 1, act)
    stage_out = []
    for i, (c, n) in enumerate(zip(widths, depths)):
        stage_out.append(darknet._csp_stage(b, c, n, act, first=(i == 0)))
    c5 = widths[-1] // 2
    p5 = darknet._csp_spp(b, c5, act, neck_n)
    b.conv(c5 // 2, 1, 1, act); b.upsample()
    b.route([stage_out[-2]]); b.conv(c5 // 2, 1, 1, act); b.route([-1, -3])
    p4 = darknet._csp_up(b, c5 // 2, neck_n, act)
    b.conv(c5 // 4, 1, 1, act); b.upsample()
    b.route([stage_out[-3]]); b.conv(c5 // 4, 1, 1, act); b.route([-1, -3])
    p3 = darknet._csp_up(b, c5 // 4, neck_n, act)
    b.conv(c5 // 2, 3, 1, act); b.conv(out_c, 1, 1, 'logistic', bn=0); b.yolo()
    b.route([p3]); b.conv(c5 // 2, 3, 2, act); b.route([-1, p4])
    n4 = darknet._csp_up(b, c5 // 2, neck_n, act)
    b.conv(c5, 3, 1, act); b.conv(out_c, 1, 1, 'logistic', bn=0); b.yolo()
    b.route([n4]); b.conv(c5, 3, 2, act); b.route([-1, p5])
    darknet._csp_up(b, c5, neck_n, act)
    b.conv(c5 * 2, 3, 1, act); b.conv(out_c, 1, 1, 'logistic', bn=0); b.yolo()
    return b.layers


@pytest.mark.parametrize("nc,apn", [(1, 3), (1, 4), (80, 3)])
def test_generalised_scaled_yolov4_keeps_the_csp_and_p5_layer_lists(nc, apn):
    assert darknet.yolov4_csp(nc, apn) == _scaled_yolov4_three_levels([1, 2, 8, 8, 4], [64, 128, 256, 512, 1024], 2,
                                                                      nc, apn)
    assert darknet.yolov4_p5(nc, apn) == _scaled_yolov4_three_levels([1, 3, 15, 15, 7], [64, 128, 256, 512, 1024], 3,
                                                                     nc, apn)


@pytest.mark.parametrize("name", ALL)
def test_head_shapes_match_the_descriptor(name):
    m = models.YOLO.get_model(name)
    _, H, W = m.INPUT_SHAPE
    got = darknet.head_shapes(_layers(m), H, W)
    want = [((5 + m.NUM_CLASSES) * (len(a) // 2), H // f, W // f) for f, a in zip(m.LAYER_FACTORS, m.ANCHORS)]
    assert got == want
    check_heads(m, got)


# ------------------------------------------------------------------------------------------------ descriptors
@pytest.mark.parametrize("name", NEW)
def test_descriptors_equal_the_reference_registry(name):
    """Every value of the reference's class (fastmot/models/yolo.py at the line given in REFERENCE), except that
    YOLOv3 and YOLOv3SPP get a third SCALES entry of 1.0 (Darknet's default scale_x_y): the reference lists two for
    three heads, which its own add_plugin rejects."""
    line, nc, lb, newc, shape, factors, scales, anchors = REFERENCE[name]
    m = models.YOLO.get_model(name)
    assert (m.NUM_CLASSES, m.LETTERBOX, m.NEW_COORDS, m.INPUT_SHAPE, m.LAYER_FACTORS, m.ANCHORS) == \
        (nc, lb, newc, shape, factors, anchors), line
    if name in ('YOLOv3', 'YOLOv3SPP'):
        assert m.SCALES == scales + [1.0]
    else:
        assert m.SCALES == scales
    assert m.CFG in darknet.BUILDERS


def test_eleven_reference_models_are_registered():
    for name in ALL:
        m = models.YOLO.get_model(name)
        check_heads(m)


def test_max_anchors_matches_the_header():
    hdr = open(os.path.join(ROOT, "include", "fastmot_b200.h")).read()
    assert int(re.search(r"#define FM_MAX_ANCHORS (\d+)", hdr).group(1)) == MAX_ANCHORS


def _custom(base, **kw):
    return type('Custom' + base.__name__, (base,), kw)


def test_head_table_validation_rejects_malformed_descriptors():
    v3 = models.YOLO.get_model('YOLOv3')
    shapes = darknet.head_shapes(_layers(v3), 416, 416)
    with pytest.raises(ValueError, match=r"CustomYOLOv3: SCALES has 2 entries for 3 \[yolo\] layers"):
        check_heads(_custom(v3, SCALES=[1.0, 1.0]), shapes)          # the reference's own YOLOv3 table
    with pytest.raises(ValueError, match="CustomYOLOv3: SCALES has 2 entries for 3 LAYER_FACTORS"):
        check_heads(_custom(v3, SCALES=[1.0, 1.0]))
    with pytest.raises(ValueError, match=r"head 2 has a 52x52 grid in the graph, but .* gives 26x26"):
        check_heads(_custom(v3, LAYER_FACTORS=[32, 16, 16]), shapes)
    with pytest.raises(ValueError, match="LAYER_FACTORS has 2 entries for 3"):
        check_heads(_custom(v3, LAYER_FACTORS=[32, 16]), shapes)
    with pytest.raises(ValueError, match=r"head 0 has 18 channels in the graph, but .* = 24"):
        check_heads(_custom(v3, ANCHORS=[[10, 13, 16, 30, 33, 23, 40, 40]] + v3.ANCHORS[1:]), shapes)
    seven = [[i + 1, i + 2] * 7 for i in range(3)]
    with pytest.raises(ValueError, match="head 0 lists 14 anchor values; a head takes 1 to 6"):
        check_heads(_custom(v3, ANCHORS=seven))
    p6 = models.YOLO.get_model('YOLOv4P6')
    with pytest.raises(ValueError, match="CustomYOLOv4P6: ANCHORS has 3 entries for 4"):
        check_heads(_custom(p6, ANCHORS=p6.ANCHORS[:3]), darknet.head_shapes(_layers(p6), 1280, 1280))


def test_build_yolo_engine_validates_before_building():
    """The engine builder checks the table against the graph before it allocates anything (no device needed to fail)."""
    from fastmot_b200.engine import build_yolo_engine
    bad = _custom(models.YOLO.get_model('YOLOv3Tiny'), SCALES=[1.0])
    with pytest.raises(ValueError, match="CustomYOLOv3Tiny: SCALES has 1 entries for 2"):
        build_yolo_engine(bad)


# ------------------------------------------------------------------------------------------------ Darknet files
@pytest.mark.parametrize("name", NEW)
def test_cfg_and_weights_round_trip(name, tmp_path):
    m = models.YOLO.get_model(name)
    layers = _layers(m)
    _, H, W = m.INPUT_SHAPE
    net, back = darknet.parse_cfg(darknet.to_cfg(layers, W, H))
    assert (net['width'], net['height']) == (W, H)
    assert back == layers
    weights = darknet.synthetic_weights(layers, 3, head_obj_bias=-4.0, num_classes=m.NUM_CLASSES, calibrate=False)
    path = str(tmp_path / "net.weights")
    darknet.save_weights(path, layers, weights, 3)
    loaded = darknet.load_weights(path, back, 3)
    assert sorted(loaded) == sorted(weights)
    for i, (w, b) in weights.items():
        assert loaded[i][0].shape == w.shape
        np.testing.assert_allclose(loaded[i][0], w, rtol=3e-7, atol=1e-9)
        np.testing.assert_array_equal(loaded[i][1], b)


# ------------------------------------------------------------------------------------------------ float64 executor
@pytest.mark.parametrize("cfg", ['yolov3', 'yolov3-spp', 'yolov3-tiny', 'yolov4x-mish', 'yolov4-csp-swish',
                                 'yolov4-csp-x-swish', 'yolov4-p6'])
def test_float64_darknet_executor_matches_oracle(cfg):
    """As tests/test_yolo64.py does for the first four models, at a 128 x 64 input (P6's stride-64 grid is 2 x 1)."""
    from oracle import nets, nets64 as R
    layers = darknet.BUILDERS[cfg](anchors_per_head=4 if cfg == 'yolov4-p6' else 3)
    w = darknet.synthetic_weights(layers, 3, head_obj_bias=-3.0)
    w64 = {i: (a.astype(np.float64), b.astype(np.float64)) for i, (a, b) in w.items()}
    x = torch.rand(1, 3, 128, 64, generator=torch.Generator().manual_seed(0), dtype=torch.float64)
    got = R.run_darknet64(layers, w, x)
    want = nets.run_darknet(layers, w64, x)
    assert len(got) == len(want) == len(darknet.head_shapes(layers, 128, 64))
    for g, h in zip(got, want):
        assert g.shape == h.shape
        assert float((g - h).abs().max() / h.abs().max()) < 1e-5
