"""Darknet network descriptions for the detector engine.

The reference runs YOLO through TensorRT engines converted from Darknet cfg/weights by scripts/yolo2onnx.py; the
supported layer vocabulary is that script's (`convolutional`, `maxpool`, `route` incl. channel groups, `shortcut`,
`upsample`, `yolo`; scripts/yolo2onnx.py:100-101, 558-870).  This module provides
  * `parse_cfg(text)`      — Darknet .cfg text -> layer list (same fields DarkNetParser keeps, yolo2onnx.py:86-205)
  * `load_weights(...)`    — Darknet .weights reader in the converter's order (yolo2onnx.py:283-400): 5 x int32
                             header (major, minor, revision, seen[64-bit if major*10+minor >= 2]), then per conv:
                             BN bias, scale, mean, var (or conv bias) followed by the conv weights [out][in][kh][kw]
  * builders for the eleven models named by fastmot/models/yolo.py (YOLOv3 / -SPP / -tiny, YOLOv4 / -tiny, and the
    Scaled-YOLOv4 csp / csp-swish / csp-x-swish / x-mish / p5 / p6).  The official cfg
    files are not in the reference tree (downloaded by scripts/download_models.sh), so the builders restate the
    published architectures; `count_flops` reports the Darknet "BFLOPs" figure for a sanity check.
  * `synthetic_weights(...)` — seeded He-normal weights with folded BN (there are no trained weights offline).
"""
import functools

import numpy as np

ACTS = {'linear': 0, 'leaky': 1, 'mish': 2, 'swish': 3, 'logistic': 4, 'relu': 5}


# ------------------------------------------------------------------------------------------------ cfg parser
def parse_cfg(text):
    layers, cur = [], None
    for raw in text.splitlines():
        line = raw.split('#')[0].strip()
        if not line:
            continue
        if line.startswith('['):
            if cur is not None:
                layers.append(cur)
            cur = {'type': line.strip('[]').strip()}
            continue
        k, v = (s.strip() for s in line.split('=', 1))
        if k in ('layers', 'anchors', 'mask'):
            cur[k] = [float(x) if '.' in x else int(x) for x in v.replace(' ', '').split(',') if x]
        else:
            try:
                cur[k] = int(v)
            except ValueError:
                try:
                    cur[k] = float(v)
                except ValueError:
                    cur[k] = v
    if cur is not None:
        layers.append(cur)
    net = layers[0] if layers and layers[0]['type'] == 'net' else {}
    return net, [l for l in layers if l['type'] != 'net']


# ------------------------------------------------------------------------------------------------ builders
class _B:
    def __init__(self):
        self.layers = []

    def conv(self, filters, size=3, stride=1, act='leaky', bn=1):
        self.layers.append(dict(type='convolutional', filters=filters, size=size, stride=stride, pad=1,
                                batch_normalize=bn, activation=act))
        return len(self.layers) - 1

    def route(self, layers, groups=1, group_id=0):
        d = dict(type='route', layers=list(layers))
        if groups > 1:
            d.update(groups=groups, group_id=group_id)
        self.layers.append(d)
        return len(self.layers) - 1

    def shortcut(self, frm):
        self.layers.append(dict(type='shortcut', activation='linear', **{'from': frm}))
        return len(self.layers) - 1

    def maxpool(self, size, stride):
        self.layers.append(dict(type='maxpool', size=size, stride=stride))
        return len(self.layers) - 1

    def upsample(self):
        self.layers.append(dict(type='upsample', stride=2))
        return len(self.layers) - 1

    def yolo(self):
        self.layers.append(dict(type='yolo'))
        return len(self.layers) - 1


def yolov4_tiny(num_classes=1, anchors_per_head=3):
    b = _B()
    out_c = anchors_per_head * (5 + num_classes)
    b.conv(32, 3, 2); b.conv(64, 3, 2)
    for c in (64, 128, 256):
        x = b.conv(c, 3, 1)
        b.route([-1], groups=2, group_id=1)
        y = b.conv(c // 2, 3, 1)
        b.conv(c // 2, 3, 1)
        b.route([-1, -2])
        z = b.conv(c, 1, 1)
        b.route([x, z])
        b.maxpool(2, 2)
        last_z = z
    b.conv(512, 3, 1)
    p = b.conv(256, 1, 1)
    b.conv(512, 3, 1)
    b.conv(out_c, 1, 1, 'linear', bn=0)
    b.yolo()
    b.route([p])
    b.conv(128, 1, 1)
    b.upsample()
    b.route([-1, last_z])
    b.conv(256, 3, 1)
    b.conv(out_c, 1, 1, 'linear', bn=0)
    b.yolo()
    return b.layers


def _csp_stage(b, c, n, act, first=False):
    """Downsample conv + CSP block with n residual units (Scaled-YOLOv4 backbone stage)."""
    b.conv(c, 3, 2, act)
    if first:
        b.conv(c // 2, 1, 1, act)
        b.conv(c, 3, 1, act)
        b.shortcut(-3)
        return len(b.layers) - 1
    h = c // 2
    b.conv(h, 1, 1, act)             # split 1 (bypass)
    b.route([-2])
    b.conv(h, 1, 1, act)             # split 2
    for _ in range(n):
        b.conv(h, 1, 1, act)
        b.conv(h, 3, 1, act)
        b.shortcut(-3)
    b.conv(h, 1, 1, act)
    b.route([-1, -(3 * n + 4)])
    return b.conv(c, 1, 1, act)


def _csp_up(b, c, n, act):
    """CSP block without shortcuts used in the PAN neck (c = hidden width, output c)."""
    b.conv(c, 1, 1, act)
    b.route([-2])
    b.conv(c, 1, 1, act)
    for _ in range(n):
        b.conv(c, 1, 1, act)
        b.conv(c, 3, 1, act)
    b.route([-1, -(2 * n + 3)])
    return b.conv(c, 1, 1, act)


def _csp_spp(b, c, act, n=1):
    b.conv(c, 1, 1, act)             # bypass
    b.route([-2])
    b.conv(c, 1, 1, act)
    b.conv(c, 3, 1, act)
    b.conv(c, 1, 1, act)
    b.maxpool(5, 1); b.route([-2]); b.maxpool(9, 1); b.route([-4]); b.maxpool(13, 1)
    b.route([-1, -3, -5, -6])
    b.conv(c, 1, 1, act)
    b.conv(c, 3, 1, act)
    for _ in range(n - 1):
        b.conv(c, 1, 1, act)
        b.conv(c, 3, 1, act)
    b.route([-1, -(13 + 2 * (n - 1))])
    return b.conv(c, 1, 1, act)


def _scaled_yolov4(depths, widths, neck_n, num_classes, anchors_per_head, act='mish', levels=3, stem=32):
    """Scaled-YOLOv4 (Wang, Bochkovskiy, Liao, CVPR 2021; models/yolov4-*.yaml of WongKinYiu/ScaledYOLOv4): a stem
    conv, one CSP stage per entry of widths / depths (each halves the resolution), an SPP-CSP block on the last stage
    and a PAN neck over the last `levels` stages (level l has width widths[l] / 2, heads twice that).  Heads run finest
    first (strides 8, 16, ...)."""
    b = _B()
    out_c = anchors_per_head * (5 + num_classes)
    b.conv(stem, 3, 1, act)
    stage_out = []
    for i, (c, n) in enumerate(zip(widths, depths)):
        stage_out.append(_csp_stage(b, c, n, act, first=(i == 0)))
    stage_out = stage_out[-levels:]
    nw = [c // 2 for c in widths[-levels:]]
    td = [None] * (levels - 1) + [_csp_spp(b, nw[-1], act, neck_n)]
    for l in range(levels - 2, -1, -1):           # top-down
        b.conv(nw[l], 1, 1, act); b.upsample()
        b.route([stage_out[l]]); b.conv(nw[l], 1, 1, act); b.route([-1, -3])
        td[l] = _csp_up(b, nw[l], neck_n, act)
    prev = td[0]
    for l in range(levels):                       # heads + bottom-up
        if l:
            b.route([prev]); b.conv(nw[l], 3, 2, act); b.route([-1, td[l]])
            prev = _csp_up(b, nw[l], neck_n, act)
        b.conv(2 * nw[l], 3, 1, act); b.conv(out_c, 1, 1, 'logistic', bn=0); b.yolo()
    return b.layers


def yolov4_csp(num_classes=1, anchors_per_head=3, act='mish'):
    """YOLOv4-CSP (ScaledYOLOv4 models/yolov4-csp.yaml; Darknet yolov4-csp.cfg, and yolov4-csp-swish.cfg with
    act='swish')."""
    return _scaled_yolov4([1, 2, 8, 8, 4], [64, 128, 256, 512, 1024], 2, num_classes, anchors_per_head, act)


def yolov4_p5(num_classes=1, anchors_per_head=4):
    return _scaled_yolov4([1, 3, 15, 15, 7], [64, 128, 256, 512, 1024], 3, num_classes, anchors_per_head)


def yolov4_csp_x(num_classes=1, anchors_per_head=3, act='mish'):
    """YOLOv4-CSP-x: yolov4-csp at width multiple 1.25 and depth multiple 1.33 (ScaledYOLOv4 models/yolov4-csp-x.yaml;
    the Darknet yolov4x-mish.cfg / yolov4-csp-x-swish.cfg): stem 40, stages 80 ... 1280 with depths 1 / 3 / 11 / 11 / 5,
    neck depth 3."""
    return _scaled_yolov4([1, 3, 11, 11, 5], [80, 160, 320, 640, 1280], 3, num_classes, anchors_per_head, act,
                          stem=40)


def yolov4_p6(num_classes=1, anchors_per_head=4):
    """YOLOv4-P6 (ScaledYOLOv4 models/yolov4-p6.yaml, Darknet yolov4-p6.cfg): the P5 backbone plus a sixth stage
    (1024 wide, 7 units) at stride 64, the SPP-CSP block on it and a four-level neck (widths 128 / 256 / 512 / 512),
    four heads at strides 8 / 16 / 32 / 64."""
    return _scaled_yolov4([1, 3, 15, 15, 7, 7], [64, 128, 256, 512, 1024, 1024], 3, num_classes, anchors_per_head,
                          levels=4)


def _darknet53(b):
    """Darknet-53 (Redmon & Farhadi, "YOLOv3: An Incremental Improvement", 2018; cfg/yolov3.cfg layers 0-74): returns
    the layer indices of its five stage outputs (strides 2 ... 32)."""
    b.conv(32, 3, 1)
    outs = []
    for c, n in zip((64, 128, 256, 512, 1024), (1, 2, 8, 8, 4)):
        b.conv(c, 3, 2)
        for _ in range(n):
            b.conv(c // 2, 1, 1); b.conv(c, 3, 1); b.shortcut(-3)
        outs.append(len(b.layers) - 1)
    return outs


def _yolov3(num_classes, anchors_per_head, spp):
    b = _B()
    out_c = anchors_per_head * (5 + num_classes)
    outs = _darknet53(b)
    x = None
    for lvl, c in enumerate((512, 256, 128)):     # heads coarsest first (strides 32, 16, 8)
        if lvl:
            b.route([x]); b.conv(c, 1, 1); b.upsample(); b.route([-1, outs[4 - lvl]])
        b.conv(c, 1, 1); b.conv(2 * c, 3, 1); b.conv(c, 1, 1)
        if spp and not lvl:
            b.maxpool(5, 1); b.route([-2]); b.maxpool(9, 1); b.route([-4]); b.maxpool(13, 1)
            b.route([-1, -3, -5, -6])
            b.conv(c, 1, 1)
        b.conv(2 * c, 3, 1)
        x = b.conv(c, 1, 1)
        b.conv(2 * c, 3, 1)
        b.conv(out_c, 1, 1, 'linear', bn=0)
        b.yolo()
    return b.layers


def yolov3(num_classes=1, anchors_per_head=3):
    """YOLOv3 (cfg/yolov3.cfg of pjreddie/darknet): Darknet-53 + an FPN of three heads, 107 layers."""
    return _yolov3(num_classes, anchors_per_head, spp=False)


def yolov3_spp(num_classes=1, anchors_per_head=3):
    """YOLOv3-SPP (cfg/yolov3-spp.cfg of pjreddie/darknet): YOLOv3 with a 5 / 9 / 13 max-pool SPP block in the
    stride-32 head, 114 layers."""
    return _yolov3(num_classes, anchors_per_head, spp=True)


def yolov3_tiny(num_classes=1, anchors_per_head=3):
    """YOLOv3-tiny (cfg/yolov3-tiny.cfg of pjreddie/darknet): six 3x3 convs each followed by a 2x2 max-pool (the last
    one at stride 1), two heads (strides 32, 16), 24 layers."""
    b = _B()
    out_c = anchors_per_head * (5 + num_classes)
    for c in (16, 32, 64, 128, 256, 512):
        b.conv(c, 3, 1)
        b.maxpool(2, 1 if c == 512 else 2)
    b.conv(1024, 3, 1)
    p = b.conv(256, 1, 1)
    b.conv(512, 3, 1)
    b.conv(out_c, 1, 1, 'linear', bn=0)
    b.yolo()
    b.route([p])
    b.conv(128, 1, 1)
    b.upsample()
    b.route([-1, 8])                              # the 256-wide conv at stride 16
    b.conv(256, 3, 1)
    b.conv(out_c, 1, 1, 'linear', bn=0)
    b.yolo()
    return b.layers


def yolov4(num_classes=2, anchors_per_head=3):
    """YOLOv4 (CSPDarknet53-mish + SPP + PANet-leaky), the CrowdHuman model of fastmot/models/yolo.py:154-163."""
    b = _B()
    out_c = anchors_per_head * (5 + num_classes)
    b.conv(32, 3, 1, 'mish')
    outs = []
    for i, (c, n) in enumerate(zip([64, 128, 256, 512, 1024], [1, 2, 8, 8, 4])):
        b.conv(c, 3, 2, 'mish')
        h = c if i == 0 else c // 2
        b.conv(h, 1, 1, 'mish'); b.route([-2]); b.conv(h, 1, 1, 'mish')
        for _ in range(n):
            b.conv(c // 2, 1, 1, 'mish'); b.conv(h, 3, 1, 'mish'); b.shortcut(-3)
        b.conv(h, 1, 1, 'mish'); b.route([-1, -(3 * n + 4)])
        outs.append(b.conv(c, 1, 1, 'mish'))
    a = 'leaky'
    b.conv(512, 1, 1, a); b.conv(1024, 3, 1, a); b.conv(512, 1, 1, a)
    b.maxpool(5, 1); b.route([-2]); b.maxpool(9, 1); b.route([-4]); b.maxpool(13, 1); b.route([-1, -3, -5, -6])
    b.conv(512, 1, 1, a); b.conv(1024, 3, 1, a); p5 = b.conv(512, 1, 1, a)
    b.conv(256, 1, 1, a); b.upsample(); b.route([outs[3]]); b.conv(256, 1, 1, a); b.route([-1, -3])
    for _ in range(2):
        b.conv(256, 1, 1, a); b.conv(512, 3, 1, a)
    p4 = b.conv(256, 1, 1, a)
    b.conv(128, 1, 1, a); b.upsample(); b.route([outs[2]]); b.conv(128, 1, 1, a); b.route([-1, -3])
    for _ in range(2):
        b.conv(128, 1, 1, a); b.conv(256, 3, 1, a)
    p3 = b.conv(128, 1, 1, a)
    b.conv(256, 3, 1, a); b.conv(out_c, 1, 1, 'linear', bn=0); b.yolo()
    b.route([p3]); b.conv(256, 3, 2, a); b.route([-1, p4])
    for _ in range(2):
        b.conv(256, 1, 1, a); b.conv(512, 3, 1, a)
    n4 = b.conv(256, 1, 1, a)
    b.conv(512, 3, 1, a); b.conv(out_c, 1, 1, 'linear', bn=0); b.yolo()
    b.route([n4]); b.conv(512, 3, 2, a); b.route([-1, p5])
    for _ in range(2):
        b.conv(512, 1, 1, a); b.conv(1024, 3, 1, a)
    b.conv(512, 1, 1, a)
    b.conv(1024, 3, 1, a); b.conv(out_c, 1, 1, 'linear', bn=0); b.yolo()
    return b.layers


BUILDERS = {'yolov4-tiny': yolov4_tiny, 'yolov4-csp': yolov4_csp, 'yolov4-p5': yolov4_p5, 'yolov4': yolov4,
            'yolov3': yolov3, 'yolov3-spp': yolov3_spp, 'yolov3-tiny': yolov3_tiny,
            'yolov4x-mish': yolov4_csp_x, 'yolov4-csp-swish': functools.partial(yolov4_csp, act='swish'),
            'yolov4-csp-x-swish': functools.partial(yolov4_csp_x, act='swish'), 'yolov4-p6': yolov4_p6}


def head_shapes(layers, in_h, in_w):
    """(c, h, w) of every [yolo] layer's input, in graph order, for an in_h x in_w network input."""
    res, shapes = infer_shapes(layers, 3, in_h, in_w)
    return [shapes[i] for i, l in enumerate(res) if l['type'] == 'yolo']


# ------------------------------------------------------------------------------------------------ shape inference
def infer_shapes(layers, in_c, in_h, in_w):
    """Returns per-layer (c, h, w) and resolves route/shortcut indices to absolute layer numbers (in place copy)."""
    shapes, resolved = [], []
    for i, l in enumerate(layers):
        l = dict(l)
        t = l['type']
        pc, ph, pw = shapes[-1] if shapes else (in_c, in_h, in_w)
        if t == 'convolutional':
            s = l.get('stride', 1)
            shapes.append((l['filters'], (ph + s - 1) // s, (pw + s - 1) // s))
            l['in_c'] = pc
        elif t == 'maxpool':
            s = l['stride']
            shapes.append((pc, (ph + s - 1) // s, (pw + s - 1) // s))
        elif t == 'upsample':
            shapes.append((pc, ph * l['stride'], pw * l['stride']))
        elif t == 'shortcut':
            f = l['from']
            l['from_abs'] = f if f >= 0 else i + f
            shapes.append((pc, ph, pw))
        elif t == 'route':
            srcs = [x if x >= 0 else i + x for x in l['layers']]
            l['layers_abs'] = srcs
            g = l.get('groups', 1)
            cs = [shapes[s][0] // g for s in srcs]
            shapes.append((sum(cs), shapes[srcs[0]][1], shapes[srcs[0]][2]))
        elif t == 'yolo':
            shapes.append((pc, ph, pw))
        else:
            raise NotImplementedError(f"Darknet layer type {t}")
        resolved.append(l)
    return resolved, shapes


def count_flops(layers, in_c, in_h, in_w):
    """Darknet's BFLOPs convention: 2 * Cin * k^2 * Cout * Hout * Wout summed over conv layers."""
    res, shapes = infer_shapes(layers, in_c, in_h, in_w)
    total = 0
    for l, (c, h, w) in zip(res, shapes):
        if l['type'] == 'convolutional':
            total += 2 * l['in_c'] * l['size'] ** 2 * c * h * w
    return total


# ------------------------------------------------------------------------------------------------ weights
def synthetic_weights(layers, in_c, seed_base=1000, head_obj_bias=None, num_classes=1, calibrate=True, head_gain=1.0):
    """Seeded He-normal conv weights (seed = seed_base + layer index, SURVEY.md §8d) with BN folded.
    Returns {layer_index: (weight [out][kh][kw][in] float32, bias float32[out])}.
    head_obj_bias: if set, the objectness bias of every head conv (the conv right before a [yolo] layer) is
    initialised to it — the usual detection-prior init — so random weights give a sparse, trained-like candidate set.
    head_gain: scale of the head convs' weights after calibration (< 1 shrinks the logit variance real frames produce
    in the deep models, so that the objectness prior, not noise, decides how many candidates pass conf_thresh)."""
    res, _ = infer_shapes(layers, in_c, 64, 64)
    out = {}
    for i, l in enumerate(res):
        if l['type'] != 'convolutional':
            continue
        rng = np.random.default_rng(seed_base + i)
        k, cin, cout = l['size'], l['in_c'], l['filters']
        w = rng.normal(0, np.sqrt(2.0 / (k * k * cin)), (cout, k, k, cin)).astype(np.float32)
        b = rng.normal(0, 0.02, cout).astype(np.float32)
        is_head = i + 1 < len(res) and res[i + 1]['type'] == 'yolo'
        if is_head:
            b[:] = 0
            if head_obj_bias is not None:
                info = 5 + num_classes
                b[4::info] = head_obj_bias
        out[i] = (w, b)
    if calibrate:
        from .calibrate import calibrate_darknet
        # a 4 x 4 grid at the coarsest stride at least: the channel statistics of P6's stride-64 stage taken on 2 x 2
        # pixels leave its activations past the fp16 range at 1280 (strides up to 32 calibrate at 128, as before)
        stride = 64 // min(s[1] for s in infer_shapes(layers, in_c, 64, 64)[1])
        out = calibrate_darknet(res, out, in_c, size=max(128, 4 * stride))
    if head_gain != 1.0:
        for i, l in enumerate(res):
            if l['type'] == 'convolutional' and i + 1 < len(res) and res[i + 1]['type'] == 'yolo':
                w, b = out[i]
                out[i] = ((w * np.float32(head_gain)).astype(np.float32), b)
    return out


def to_cfg(layers, width, height, channels=3):
    """Darknet .cfg text for a layer list (inverse of parse_cfg; scripts/yolo2onnx.py:86-205 reads this format).
    Layer-index references (`layers`, `from`) are written as they are stored (relative or absolute)."""
    out = ["[net]", f"width={width}", f"height={height}", f"channels={channels}", ""]
    for l in layers:
        out.append(f"[{l['type']}]")
        for k, v in l.items():
            if k == 'type' or k.endswith('_abs') or k in ('in_c', 'out_c'):
                continue
            if isinstance(v, (list, tuple)):
                v = ",".join(str(x) for x in v)
            out.append(f"{k}={v}")
        out.append("")
    return "\n".join(out)


def save_weights(path, layers, weights, in_c):
    """Writes {layer_index: (weight [out][kh][kw][in], bias)} (BN already folded) as a Darknet .weights file
    (header version 0.2.5, 64-bit `seen`; per conv: BN beta, gamma, mean, var | conv bias, then [out][in][kh][kw]
    weights -- scripts/yolo2onnx.py:283-400).  Folded weights are stored with an identity batch norm (gamma 1,
    mean 0, var 1 - eps), so load_weights() reproduces them up to one fp32 rounding of the BN scale."""
    import struct
    res, _ = infer_shapes(layers, in_c, 64, 64)
    with open(path, 'wb') as f:
        f.write(struct.pack('<iii', 0, 2, 5))
        f.write(struct.pack('<q', 0))
        for i, l in enumerate(res):
            if l['type'] != 'convolutional':
                continue
            w, b = weights[i]
            cout = w.shape[0]
            wd = np.ascontiguousarray(np.asarray(w, np.float32).transpose(0, 3, 1, 2))
            if l.get('batch_normalize', 0):
                for a in (np.asarray(b, np.float32), np.ones(cout, np.float32), np.zeros(cout, np.float32),
                          np.full(cout, 1.0 - 1e-5, np.float32)):
                    f.write(a.tobytes())
            else:
                f.write(np.asarray(b, np.float32).tobytes())
            f.write(wd.tobytes())


def load_weights(path, layers, in_c):
    """Darknet .weights -> {layer_index: (weight [out][kh][kw][in], bias)} with BN folded (eps 1e-5,
    yolo2onnx.py:419)."""
    res, _ = infer_shapes(layers, in_c, 64, 64)
    with open(path, 'rb') as f:
        major, minor, _rev = np.frombuffer(f.read(12), np.int32)
        f.read(8 if major * 10 + minor >= 2 else 4)
        data = np.frombuffer(f.read(), np.float32)
    pos = 0

    def take(n):
        nonlocal pos
        if pos + n > len(data):
            raise ValueError("weights file too short for this cfg")
        a = data[pos:pos + n]
        pos += n
        return a

    out = {}
    for i, l in enumerate(res):
        if l['type'] != 'convolutional':
            continue
        k, cin, cout = l['size'], l['in_c'], l['filters']
        if l.get('batch_normalize', 0):
            beta, gamma, mean, var = take(cout), take(cout), take(cout), take(cout)
            w = take(cout * cin * k * k).reshape(cout, cin, k, k)
            scale = gamma / np.sqrt(var + 1e-5)
            w = w * scale[:, None, None, None]
            b = beta - mean * scale
        else:
            b = take(cout)
            w = take(cout * cin * k * k).reshape(cout, cin, k, k)
        out[i] = (np.ascontiguousarray(w.transpose(0, 2, 3, 1)).astype(np.float32), b.astype(np.float32))
    return out
