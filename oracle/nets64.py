"""TEST INFRASTRUCTURE ONLY.  float64 reference of every OSNet op (models/osnet.py vocabulary) and of the fused units
the engine launches (the stem, fm_osb_streams = "S", fm_osb_merge = "G"), of the Darknet layers the detector engine
launches (conv with every activation, max-pool, upsample, route copy, shortcut) and of the head decode, each with a
per-element error bound derived from the rounding model of the kernel that computes it.

Every function takes the fp16 / fp32 values the kernel read (any torch dtype, any device; NHWC activations) and
returns (want, bound) as float64 tensors: `want` is the exact result rounded to fp16 wherever the kernel stores
fp16, and |kernel output - want| <= bound must hold element-wise.  With `q=False` nothing is rounded (the
composed executor `run_ops`, compared with oracle.nets.run_osnet).

Symbols of the rounding models: u = 2^-11 (fp16 unit roundoff), u32 = 2^-24 (fp32), eta = 2^-25 (absolute error of
one rounding into the fp16 subnormal range), K = reduction length, S|xw| = the same contraction applied to |x|, |w|.
"""
import math

import torch
import torch.nn.functional as F

from fastmot_b200.models import darknet

U16 = 2.0 ** -11
U32 = 2.0 ** -24
ETA16 = 2.0 ** -25
D = torch.float64


def _d(t):
    return torch.as_tensor(t).to(D)


def f16(v):
    """Round to fp16 (round to nearest even), back in float64."""
    return v.to(torch.float16).to(D)


def _store16(v, e_pre, q=True):
    """fp16 store of a value the kernel holds as v_k with |v_k - v| <= e_pre.  Both the kernel and the reference
    round: |fl(v_k) - fl(v)| <= |v_k - v| + u |v_k| + u |v| + 2 eta <= e_pre + u (2 |v| + e_pre) + 2 eta."""
    if not q:
        return v, e_pre
    return f16(v), e_pre + U16 * (2 * v.abs() + e_pre) + 2 * ETA16


def _nchw(x):
    return x.permute(0, 3, 1, 2)


def _nhwc(x):
    return x.permute(0, 2, 3, 1)


def _act(v, act):
    """The activations of csrc/conv_act.cuh and nn.cu (Darknet semantics), exact."""
    if act == 'linear':
        return v
    if act == 'relu':
        return v.clamp_min(0)
    if act == 'leaky':
        return torch.where(v > 0, v, 0.1 * v)
    if act == 'logistic':
        return torch.sigmoid(v)
    if act == 'swish':
        return v * torch.sigmoid(v)
    if act == 'mish':
        return v * torch.tanh(F.softplus(v))
    raise ValueError(act)


def _expf_rel(x):
    """Relative error of __expf(x) (ex2.approx and the fp32 product x log2(e)), as in gate_vector."""
    return 2.0 ** -21 + x.abs() * 2.0 ** -23


def _act_bound(v, e, act):
    """(act(v), bound) for a kernel that holds the pre-activation as v_k, |v_k - v| <= e, and applies the fp32
    activation of conv_act.cuh / nn.cu to it.  The bound is the largest slope of the activation on [v - e, v + e]
    times e, plus the activation's own rounding relative to |act(v)|:
      linear 0; relu 0 (slope 0 where v + e <= 0);
      leaky   slope 0.1 where v + e <= 0; the product 0.1f * v: the constant 0.1f (off by 1.5e-8 relative) and
              one rounding, 2 u32;
      logistic 1 / (1 + __expf(-v)): slope <= 1/4; the relative error d of __expf(-v) reaches 1 / (1 + n) damped
              by n / (1 + n) <= 1; the add and the (IEEE or __fdividef 2-ulp) division: d + 4 u32;
      swish   v / (1 + __expf(-v)): slope <= 1.1 (max 1.0998 at v ~ 2.4); d + 4 u32;
      mish    v r, r = t / (t + 2), t = n (n + 2), n = __expf(min(v, 20)): slope <= 1.1 (max 1.089 at v ~ 1.2);
              d ln r / d ln n <= 1, so r inherits the relative error d of n; t (2 roundings), t + 2, __fdividef
              (2 ulp) and the product by v add 8 u32.  The clamp at v = 20 changes r by < 1e-16 relative.  nn.cu's
              SIMT form v tanh(log1p(n)) is the same function of n (log1pf 1 ulp, tanhf 2 ulp, both damped by
              slopes <= 1 in the log domain) and is inside the same bound.
    d is taken at |v| + e: the kernel's argument is v_k, not v."""
    y = _act(v, act)
    if act == 'linear':
        return y, e
    if act == 'relu':
        return y, torch.where(v + e > 0, e, torch.zeros_like(e))
    if act == 'leaky':
        return y, torch.where(v + e > 0, e, 0.1 * e) + 2 * U32 * y.abs()
    if act == 'logistic':
        return y, 0.25 * e + y.abs() * (_expf_rel(v.abs() + e) + 4 * U32)
    if act == 'swish':
        return y, 1.1 * e + y.abs() * (_expf_rel(v.abs() + e) + 4 * U32)
    if act == 'mish':
        return y, 1.1 * e + y.abs() * (_expf_rel((v.abs() + e).clamp_max(20.0)) + 8 * U32)
    raise ValueError(act)


# ------------------------------------------------------------------------------------------------- single ops
def conv(x, w, b, stride=1, pad=0, act='linear', res=None, res_first=True, q=True):
    """Dense conv, NHWC: x (n, h, w, cin), w (cout, k, k, cin), b (cout), optional residual (n, ho, wo, cout).
    act(conv + b + res) when res_first (FM_ACT_AFTER_RESIDUAL, OSNet conv3), else act(conv + b) + res (the Darknet
    order of a shortcut fused into the conv's epilogue).
    Model (wgmma or SIMT, fp32 accumulation, fp16 store):
        pre-activation u |acc| + K u32 S|xw| + 3 u32 (|acc| + |b| + |res|), through the activation (_act_bound),
        + u32 |out| for a residual added after it, then the fp16 store (_store16).
    `acc` is the pre-bias sum: the staged epilogue rounds it to fp16 before adding the bias (conv_tc.cu
    epilogue_staged, conv_tma.cu S == 1); the other epilogues add in fp32, for which the term is merely loose."""
    x, w, b = _d(x), _d(w), _d(b)
    k = w.shape[1]
    wt = w.permute(0, 3, 1, 2)
    acc = _nhwc(F.conv2d(_nchw(x), wt, None, stride=stride, padding=pad))
    sabs = _nhwc(F.conv2d(_nchw(x.abs()), wt.abs(), None, stride=stride, padding=pad))
    r = torch.zeros_like(acc) if res is None else _d(res)
    kk = k * k * x.shape[-1]
    e = U16 * acc.abs() + kk * U32 * sabs + 3 * U32 * (acc.abs() + b.abs() + r.abs())
    v = acc + b
    if res_first:
        v, e = _act_bound(v + r, e, act)
    else:
        v, e = _act_bound(v, e, act)
        if res is not None:
            v = v + r
            e = e + U32 * v.abs()
    return _store16(v, e, q)


def dw(x, w, b, act='relu', model='fp32', q=True):
    """Depthwise 3x3 s1 p1 + bias + act, NHWC: x (n, h, w, c), w (9, c) (tap-major), b (c).
    Models of the kernels that compute it:
      'fp32'   (nn.cu dwconv3_kernel, nn_vec.cu dwconv3_vec / _vec4): fp32 FMA chain from the bias,
               10 u32 (S|xw| + |b|);
      'rows3'  (nn_vec.cu dwconv3_tile): the three taps of a window row in packed fp16 (HMUL2 + 2 HFMA2, three
               roundings of partial sums bounded by that row's S|xw|), rows and bias summed in fp32:
               3 u S|xw| + 9 eta + 4 u32 (S|xw| + |b|);
      'chain9' (osnet_fused.cu, kernel S): bias rounded to fp16, then nine HFMA2 from it: ten fp16 roundings of
               partial sums bounded by |b| + S|xw|:  10 u (|b| + S|xw|) + 10 eta."""
    x, w, b = _d(x), _d(w), _d(b)
    c = x.shape[-1]
    wt = w.t().reshape(c, 1, 3, 3)
    acc = _nhwc(F.conv2d(_nchw(x), wt, None, padding=1, groups=c))
    sabs = _nhwc(F.conv2d(_nchw(x.abs()), wt.abs(), None, padding=1, groups=c))
    v = _act(acc + b, act)
    if model == 'fp32':
        e = 10 * U32 * (sabs + b.abs())
    elif model == 'rows3':
        e = 3 * U16 * sabs + 9 * ETA16 + 4 * U32 * (sabs + b.abs())
    elif model == 'chain9':
        e = 10 * U16 * (sabs + b.abs()) + 10 * ETA16
    else:
        raise ValueError(model)
    return _store16(v, e, q)


def maxpool3s2(x, q=True):
    """3x3 / stride 2 / pad 1 max-pool: exact (a max of fp16 values is stored unchanged)."""
    x = _d(x)
    want = _nhwc(F.max_pool2d(_nchw(x), 3, 2, 1))
    return want, torch.zeros_like(want)


def avgpool2(x, q=True):
    """2x2 average: four fp16 values summed in fp32 and scaled by 0.25 (exact): 3 u32 mean|x|, fp16 store."""
    x = _d(x)
    want = _nhwc(F.avg_pool2d(_nchw(x), 2))
    sabs = _nhwc(F.avg_pool2d(_nchw(x.abs()), 2))
    return _store16(want, 3 * U32 * sabs, q)


def gate_vector(mean, e_mean, w1, b1, w2, b2):
    """g = sigmoid(W2 relu(W1 mean + b1) + b2) in fp32 (nn.cu gate_fc_kernel, nn_vec.cu gate_fc4*_kernel) from a
    channel mean known to within e_mean.  Returns (g, bound): the FC sums propagate e_mean through |W| and add
    (K + 1) u32 (S|wx| + |b|) each; sigmoid has slope g (1 - g) <= 1/4 (+ 0.1 |da| to first order, |sigmoid''| <= 0.1);
    __expf(-a) carries a relative error <= 2^-21 + |a| 2^-23 (ex2.approx and the fp32 product a log2(e)); the
    division adds 2 u32 g."""
    mean, e_mean = _d(mean), _d(e_mean)
    w1, b1, w2, b2 = _d(w1), _d(b1), _d(w2), _d(b2)
    c, cr = w1.shape[1], w1.shape[0]
    h = (mean @ w1.t() + b1).clamp_min(0)
    e_h = e_mean @ w1.abs().t() + (c + 1) * U32 * (mean.abs() @ w1.abs().t() + b1.abs())
    a = h @ w2.t() + b2
    e_a = e_h @ w2.abs().t() + (cr + 1) * U32 * (h.abs() @ w2.abs().t() + b2.abs())
    g = torch.sigmoid(a)
    slope = g * (1 - g) + 0.1 * e_a
    e_g = slope * (e_a + 2.0 ** -21 + a.abs() * 2.0 ** -23) + 2 * U32 * g
    return g, e_g


def channel_mean(x):
    """Mean over the pixels of each crop and channel, fp32 sums of hw terms: (hw - 1) u32 mean|x| + u32 |mean|."""
    x = _d(x)
    n, h, w, c = x.shape
    m = x.mean((1, 2))
    return m, (h * w) * U32 * x.abs().mean((1, 2)) + U32 * m.abs()


def strip_mean(gap_part, hw):
    """Channel means from the per-strip sums of kernel S: gap_part (n, strips, 4, c) fp32, summed over the strips in
    fp32 and scaled by 1 / hw: strips u32 S|part| / hw + 2 u32 |mean|.  Returns (mean, bound) of shape (4, n, c)."""
    gp = _d(gap_part)
    m = gp.sum(1).permute(1, 0, 2) / hw
    e = gp.shape[1] * U32 * gp.abs().sum(1).permute(1, 0, 2) / hw + 2 * U32 * m.abs()
    return m, e


def gate(x, gw, acc=None, q=True):
    """fm_channel_gate: acc (+)= x * g(x), g from the channel means of x.  fp32 product (+ sum), fp16 store:
    |x| e_g + 2 u32 (|x g| + |acc|)."""
    x = _d(x)
    m, em = channel_mean(x)
    g, eg = gate_vector(m, em, *gw)
    y = x * g[:, None, None, :]
    a = torch.zeros_like(y) if acc is None else _d(acc)
    e = x.abs() * eg[:, None, None, :] + 2 * U32 * (y.abs() + a.abs())
    return _store16(y + a, e, q)


def gate4_apply(xs, g, eg, q=True):
    """u = sum_s x_s g_s in fp32 (four products, four sums), fp16 store: S|x_s| e_gs + 4 u32 S|x_s g_s|."""
    xs = [_d(x) for x in xs]
    u = sum(x * g[s][:, None, None, :] for s, x in enumerate(xs))
    e = sum(x.abs() * eg[s][:, None, None, :] for s, x in enumerate(xs))
    e = e + 4 * U32 * sum((x * g[s][:, None, None, :]).abs() for s, x in enumerate(xs))
    return _store16(u, e, q)


def gate4(xs, gw, q=True):
    """fm_channel_gate4 (shared gate of the four streams), gate from the channel means of each stream."""
    ms = [channel_mean(x) for x in xs]
    g, eg = gate_vector(torch.stack([m for m, _ in ms]), torch.stack([e for _, e in ms]), *gw)
    return gate4_apply(xs, g, eg, q)


def gate4_pooled(xs, gap_part, gw, q=True):
    """fm_channel_gate4_pooled: the same, gate from the strip sums kernel S left behind."""
    n, h, w, c = xs[0].shape
    m, em = strip_mean(gap_part, h * w)
    g, eg = gate_vector(m, em, *gw)
    return gate4_apply(xs, g, eg, q)


def add_relu(a, b, q=True):
    """relu(a + b) in fp32 (exact for fp16 operands up to one rounding), fp16 store."""
    v = (_d(a) + _d(b)).clamp_min(0)
    return _store16(v, U32 * v.abs(), q)


def gap(x, q=True):
    """Global average pool to fp32 (nn.cu gap_kernel / nn_vec.cu gap_vec)."""
    m, e = channel_mean(x)
    return m, e


def fc(x, w, b, q=True):
    """fm_fc_norm: y = relu(W x + b) in fp32 (cin + 1) u32 (S|wx| + |b|), then y / ||y||:
    |y_k / ||y_k|| - y / ||y||| <= (e_y + |out| ||e_y||) / (||y|| - ||e_y||) + (cout + 4) u32 |out|."""
    x, w, b = _d(x), _d(w), _d(b)
    y = (x @ w.t() + b).clamp_min(0)
    e_y = (x.shape[1] + 1) * U32 * (x.abs() @ w.abs().t() + b.abs())
    nrm = y.norm(dim=1, keepdim=True)
    out = y / nrm
    en = e_y.norm(dim=1, keepdim=True)
    e = (e_y + out.abs() * en) / (nrm - en) + (w.shape[0] + 4) * U32 * out.abs()
    return out, e


# ------------------------------------------------------------------------------------------------- Darknet ops
def maxpool(x, size, stride, q=True):
    """Darknet max-pool, NHWC, same-upper padding with -inf (out = ceil(in / stride), the smaller half of the padding
    on top / left; oracle.nets._same_upper_pool).  Exact: a max of fp16 values is stored unchanged."""
    x = _d(x)
    h, w = x.shape[1:3]
    ho, wo = -(-h // stride), -(-w // stride)
    ph, pw = max((ho - 1) * stride + size - h, 0), max((wo - 1) * stride + size - w, 0)
    xp = F.pad(_nchw(x), (pw // 2, pw - pw // 2, ph // 2, ph - ph // 2), value=float('-inf'))
    want = _nhwc(F.max_pool2d(xp, size, stride))
    return want, torch.zeros_like(want)


def upsample(x, stride=2, q=True):
    """Nearest upsample, NHWC: a copy (exact)."""
    x = _d(x)
    want = x.repeat_interleave(stride, 1).repeat_interleave(stride, 2)
    return want, torch.zeros_like(want)


def copy(x, q=True):
    """A route source copied into its concat slice: exact."""
    x = _d(x)
    return x, torch.zeros_like(x)


def add_act(a, b, act='linear', q=True):
    """fm_add_act_strided (Darknet shortcut): act(a + b) with an fp32 add (one rounding, u32 |a + b|), the fp32
    activation (_act_bound), fp16 store."""
    v = _d(a) + _d(b)
    v, e = _act_bound(v, U32 * v.abs(), act)
    return _store16(v, e, q)


def _f32(v):
    """Round to fp32 (round to nearest even), back in float64.  For fp32 operands, the float64 result of + - * /
    rounded once to fp32 is the correctly rounded fp32 result (53 >= 2 * 24 + 2), so a chain of _f32(a op b)
    restates a chain of fp32 _rn operations exactly."""
    return v.to(torch.float32).to(D)


def _div(a, b):
    """a / b correctly rounded: torch's CUDA division by a Python scalar multiplies by its reciprocal, which is not
    (and can move a later fp32 rounding by an ulp), so the divisor is made a tensor."""
    return a / torch.full_like(a, b)


def decode64(head, anchors, scale_x_y, input_wh, num_classes, new_coords, size=(1.0, 1.0), offset=(0.0, 0.0)):
    """csrc/detect.cu yolo_decode_filter_kernel in float64: head (A (5 + C), H, W) planar, the values the kernel read
    (fp16 or fp32).  Returns (want, bound), each (A H W, 8) in candidate order (anchor, row, column):
    columns px, py, pw, ph (pixels: scaled by `size`, minus `offset`), box_prob, class_id, cls_prob -- the dense
    row the kernel writes -- and the score box_prob * cls_prob that meets conf_thresh.

    new_coords: every step of the kernel is an fp32 _rn operation on exactly representable inputs, restated with
    _f32 after each operation: exact, bound 0.
    old coords: the sigmoids and exp go through __expf (relative error d = 2^-21 + |t| 2^-23).  The reference is the
    exact real-number result; each later fp32 operation adds u32 of its result, and the input errors propagate
    linearly (sigmoid with slope <= 1 in the relative sense, exp relative)."""
    t = _d(head)
    A = len(anchors) // 2
    C = num_classes
    _, H, W = t.shape
    t = t.reshape(A, 5 + C, H, W)
    cls = t[:, 5:]
    best = cls.max(1).values
    ids = torch.arange(C, device=t.device)[None, :, None, None]
    class_id = torch.where(cls == best[:, None], ids, C).min(1).values      # the first maximum (the strict '>' scan)
    col = torch.arange(W, dtype=D, device=t.device)[None, None, :]
    row = torch.arange(H, dtype=D, device=t.device)[None, :, None]
    aw = torch.tensor([float(a) for a in anchors[0::2]], dtype=D, device=t.device).to(torch.float32).to(D)
    ah = torch.tensor([float(a) for a in anchors[1::2]], dtype=D, device=t.device).to(torch.float32).to(D)
    aw, ah = aw[:, None, None], ah[:, None, None]
    s = float(torch.tensor(scale_x_y, dtype=torch.float32))
    iw, ih = float(input_wh[0]), float(input_wh[1])
    sw, sh = (float(torch.tensor(v, dtype=torch.float32)) for v in size)
    ox, oy = (float(torch.tensor(v, dtype=torch.float32)) for v in offset)
    hs = float(_f32(torch.tensor(s - 1.0, dtype=D))) * 0.5              # __fmul_rn(s - 1.0f, 0.5f): exact halving
    z = torch.zeros_like(best)
    if new_coords:
        f = _f32
        cls_prob, box_prob = best, t[:, 4]
        bw = f(_div(f(f(f(t[:, 2] * t[:, 2]) * 4.0) * aw), iw))
        bh = f(_div(f(f(f(t[:, 3] * t[:, 3]) * 4.0) * ah), ih))
        bx = f(_div(f(col + f(f(s * t[:, 0]) - hs)), W))
        by = f(_div(f(row + f(f(s * t[:, 1]) - hs)), H))
        bx, by = f(bx - f(bw * 0.5)), f(by - f(bh * 0.5))                 # halving is exact
        px, py = f(f(bx * sw) - ox), f(f(by * sh) - oy)
        pw, ph = f(bw * sw), f(bh * sh)
        score = f(box_prob * cls_prob)
        want = [px, py, pw, ph, box_prob, class_id.to(D), cls_prob, score]
        bound = [z] * 8
    else:
        def sig(x):
            g = torch.sigmoid(x)
            return g, g * (_expf_rel(x) + 2 * U32)       # __expf(-x), 1 + n and the IEEE division

        cls_prob, e_cls = sig(best)
        box_prob, e_box = sig(t[:, 4])
        ex, e_ex = sig(t[:, 0])
        ey, e_ey = sig(t[:, 1])
        bw = torch.exp(t[:, 2]) * aw / iw
        bh = torch.exp(t[:, 3]) * ah / ih
        e_bw = bw * (_expf_rel(t[:, 2]) + 3 * U32)        # __expf, the product by the anchor, the division
        e_bh = bh * (_expf_rel(t[:, 3]) + 3 * U32)

        def centre(cell, e, e_e, n):
            a = s * e
            ea = s * e_e + U32 * a.abs()
            a = a - hs
            ea = ea + U32 * a.abs()
            a = cell + a
            ea = ea + U32 * a.abs()
            return a / n, ea / n + U32 * (a / n).abs()

        bx, e_bx = centre(col, ex, e_ex, W)
        by, e_by = centre(row, ey, e_ey, H)
        bx, by = bx - bw / 2, by - bh / 2
        e_bx, e_by = e_bx + e_bw / 2 + 2 * U32 * bx.abs(), e_by + e_bh / 2 + 2 * U32 * by.abs()

        def pix(v, e, sc, off):
            p = v * sc
            ep = e * sc + U32 * p.abs()
            return p - off, ep + U32 * (p - off).abs()

        px, e_px = pix(bx, e_bx, sw, ox)
        py, e_py = pix(by, e_by, sh, oy)
        pw, e_pw = pix(bw, e_bw, sw, 0.0)
        ph, e_ph = pix(bh, e_bh, sh, 0.0)
        score = box_prob * cls_prob
        e_score = e_box * cls_prob + e_cls * box_prob + e_box * e_cls + U32 * score
        # the fp32 values stored: one more rounding of each (u32 relative)
        want = [px, py, pw, ph, box_prob, class_id.to(D), cls_prob, score]
        bound = [e_px, e_py, e_pw, e_ph, e_box, z, e_cls, e_score]
        bound = [e + U32 * v.abs() if j != 5 else e for j, (v, e) in enumerate(zip(want, bound))]
    want = torch.stack([v.expand(A, H, W) for v in want], -1).reshape(-1, 8)
    bound = torch.stack([v.expand(A, H, W) for v in bound], -1).reshape(-1, 8)
    return want, bound


def run_darknet64(layers, weights, x, q=False):
    """Composes the Darknet ops over a layer list of models/darknet.py (the semantics of oracle.nets.run_darknet).
    x: (1, 3, H, W).  Returns the raw head tensors [(5 + C) A, H, W] float64."""
    res, _ = darknet.infer_shapes(layers, x.shape[1], x.shape[2], x.shape[3])
    outs, heads = [], []
    cur = _nhwc(_d(x))
    for i, l in enumerate(res):
        t = l['type']
        if t == 'convolutional':
            w, b = weights[i]
            k = l['size']
            cur = conv(cur, w, b, l.get('stride', 1), k // 2 if l.get('pad', 0) else 0, l.get('activation', 'linear'),
                       q=q)[0]
        elif t == 'maxpool':
            cur = maxpool(cur, l['size'], l['stride'])[0]
        elif t == 'upsample':
            cur = upsample(cur, l['stride'])[0]
        elif t == 'shortcut':
            cur = add_act(cur, outs[l['from_abs']], l.get('activation', 'linear'), q=q)[0]
        elif t == 'route':
            g, gid = l.get('groups', 1), l.get('group_id', 0)
            parts = []
            for s_ in l['layers_abs']:
                o = outs[s_]
                c = o.shape[-1] // g
                parts.append(o[..., gid * c:(gid + 1) * c])
            cur = torch.cat(parts, -1) if len(parts) > 1 else parts[0]
        elif t == 'yolo':
            heads.append(_nchw(cur)[0].clone())
        outs.append(cur)
    return heads


# ------------------------------------------------------------------------------------------------- fused units
def stem(xb, w7, b7, q=True):
    """fm_osnet_stem: conv 7x7 / 2 / pad 3 (3 -> 64) + bias + ReLU -> fp16 -> max-pool 3x3 / 2 / pad 1.
    xb: the bordered NHWC4 input (n, H + 8, W + 8, 4) as read (the crop at +4, +4; the border is the conv padding and
    channel 3 meets zero weights).  Conv rounding model as `conv` (K = 7 * 8 * 4 slots of the A tile, fp32
    accumulation, ReLU in fp32 before the fp16 store); the pool is exact and 1-Lipschitz, so the bound is the window
    max of the conv bound."""
    xb, w7 = _d(xb), _d(w7)
    n, hb, wb, _ = xb.shape
    x = xb[:, 1:hb - 2, 1:wb - 2, :]                       # rows 2 oy + 1 .. 2 oy + 7 of the bordered image
    w = torch.zeros(w7.shape[0], 7, 7, 4, dtype=D, device=w7.device)
    w[..., :3] = w7
    wt = w.permute(0, 3, 1, 2)
    acc = _nhwc(F.conv2d(_nchw(x), wt, None, stride=2))
    sabs = _nhwc(F.conv2d(_nchw(x.abs()), wt.abs(), None, stride=2))
    b7 = _d(b7)
    v = (acc + b7).clamp_min(0)
    y, e = _store16(v, 7 * 8 * 4 * U32 * sabs + 2 * U32 * (acc.abs() + b7.abs()), q)
    want = _nhwc(F.max_pool2d(_nchw(y), 3, 2, 1))
    bound = _nhwc(F.max_pool2d(_nchw(e), 3, 2, 1))
    return want, bound


def _pw(x, w):
    return x @ w.t()


def _dwc(x, w):
    c = x.shape[-1]
    return _nhwc(F.conv2d(_nchw(x), w.t().reshape(c, 1, 3, 3), None, padding=1, groups=c))


def osb_streams(x, w1, b1, pws, dws, q=True, z=8.0):
    """Kernel S: x1 = relu(conv1x1(x) + b1) -> fp16, then four Lite-3x3 streams of 1..4 levels, each level a 1x1
    linear conv (+ bias, fp32 accumulation, fp16) and a depthwise 3x3 + bias + ReLU (HFMA2 chain, fp16); the last
    level of each stream is a tail.  x: (n, h, w, cin); w1 (mid, cin); pws / dws: ten (w, b) pairs, w (mid, mid) /
    (9, mid).  Returns the four tails as (want, bound) pairs, NHWC.

    The intermediates never leave the SM, so their rounding errors reach the tails through up to eight layers.  A
    worst-case (|W|) propagation grows by ~S|w| per layer and says nothing after three of them; instead the local
    rounding of every intermediate (bounded as in `conv` / `dw` 'chain9') is modelled as an independent zero-mean
    error, uniform within its bound (variance r^2 / 3), and its variance is carried through the squared weights
    (ReLU is 1-Lipschitz: carried unchanged).  A tail's bound is its own last rounding (worst case) plus z standard
    deviations of the propagated upstream error."""
    x = _d(x)
    n, h, w, cin = x.shape
    w1, b1 = _d(w1), _d(b1)
    acc = _pw(x, w1)
    v = (acc + b1).clamp_min(0)
    x1, r = _store16(v, cin * U32 * _pw(x.abs(), w1.abs()) + 2 * U32 * (acc.abs() + b1.abs()), q)
    var1 = r * r / 3
    tails = []
    lvl = 0
    for s in range(4):
        cur, var = x1, var1                                   # every stream starts from x1
        for j in range(s + 1):
            wp, bp = _d(pws[lvl][0]), _d(pws[lvl][1])
            wd, bd = _d(dws[lvl][0]), _d(dws[lvl][1])
            mid = wp.shape[1]
            # pointwise: fp32 accumulation of mid products + bias, fp16 store (the kernel's operand may sit z sigma
            # away from the reference's: S|xw| is taken over |x| + z sigma)
            p_acc = _pw(cur, wp)
            p, r_p = _store16(p_acc + bp, mid * U32 * _pw(cur.abs(), wp.abs()) + 2 * U32 * (p_acc.abs() + bp.abs()), q)
            var_p = _pw(var, wp * wp) + r_p * r_p / 3
            # depthwise: the fp16 HFMA2 chain of the kernel (dw model 'chain9'); zero padding outside the image.
            # Ten roundings, each of a partial sum bounded by |b| + S|xw|: variance 10 (u (|b| + S|xw|))^2 / 3
            pre = _dwc(p, wd) + bd
            sabs = _dwc(p.abs(), wd.abs())
            d, r_d = _store16(pre.clamp_min(0), 10 * U16 * (sabs + bd.abs()) + 10 * ETA16, q)
            v_d = 10 * (U16 * (sabs + bd.abs()) + ETA16) ** 2 / 3 + (U16 * (2 * d.abs()) + 2 * ETA16) ** 2 / 3
            up = _dwc(var_p, wd * wd)
            if j == s:
                tails.append((d, r_d + z * up.sqrt()))
            # ReLU: where the exact pre-activation lies below -(r_d + z sigma) the kernel stores 0 as well, and the
            # error there is exactly 0
            live = pre > -(r_d + z * up.sqrt())
            cur, var = d, torch.where(live, up + v_d, torch.zeros_like(up))
            lvl += 1
    return tails


def strip_sums(tails, strips):
    """gap_part of kernel S from the tails it stored: the per-strip channel sums of the (kernel's own) fp16 tails,
    accumulated in fp32 (one lane per pixel column, warp shuffles, four pixel quarters): rows * w u32 S|t| per
    strip.  tails: four (n, h, w, mid); returns (n, strips, 4, mid)."""
    t = torch.stack([_d(a) for a in tails], 1)                # n, 4, h, w, mid
    n, _, h, w, c = t.shape
    t = t.reshape(n, 4, strips, h // strips, w, c)
    want = t.sum((3, 4)).permute(0, 2, 1, 3)
    e = (h // strips) * w * U32 * t.abs().sum((3, 4)).permute(0, 2, 1, 3)
    return want, e


def osb_merge(tails, gap_part, gw, w3, bias, x=None, wd=None, res=None, q=True):
    """Kernel G: gate from the strip sums, u = sum_s g_s tail_s (fp32) -> fp16, then
    relu(conv3(u) [+ downsample(x)] + bias [+ res]) with fp32 accumulation and the staged fp16 epilogue.
    tails: four (n, h, w, mid); w3 (cout, mid); bias (cout) = b3 [+ b_down] as the kernel reads it; x (n, h, w, cin)
    with wd (cout, cin), or the identity res (n, h, w, cout).  The error of u reaches the output through |W3|."""
    n, h, w, mid = tails[0].shape
    m, em = strip_mean(gap_part, h * w)
    g, eg = gate_vector(m, em, *gw)
    u, e_u = gate4_apply(tails, g, eg, q)
    w3, bias = _d(w3), _d(bias)
    acc = _pw(u, w3)
    sabs = _pw(u.abs() + e_u, w3.abs())
    prop = _pw(e_u, w3.abs())
    kk = mid
    if x is not None:
        x, wd = _d(x), _d(wd)
        acc = acc + _pw(x, wd)
        sabs = sabs + _pw(x.abs(), wd.abs())
        kk += x.shape[-1]
    r = torch.zeros_like(acc) if res is None else _d(res)
    v = (acc + bias + r).clamp_min(0)
    e = prop + U16 * (acc.abs() + prop) + kk * U32 * sabs + 3 * U32 * (acc.abs() + prop + bias.abs() + r.abs())
    return _store16(v, e, q)


# ------------------------------------------------------------------------------------------------- executor
def run_ops(ops, weights, x, q=False):
    """Composes the single-op functions over an op list of models/osnet.py.  x: (n, 3, H, W) crops (NCHW, as
    oracle.nets.run_osnet takes them).  Returns the embeddings (n, feature_dim) float64."""
    bufs = {'input': _nhwc(_d(x))}
    out = None
    for op in ops:
        kind = op[0]
        if kind == 'conv':
            _, name, cin, cout, ks, stride, pad, act, src, dst = op
            w, b = weights[name]
            bufs[dst] = conv(bufs[src], w, b, stride, pad, act, q=q)[0]
        elif kind == 'dw':
            _, name, c, act, src, dst = op
            w, b = weights[name]
            bufs[dst] = dw(bufs[src], w, b, act, q=q)[0]
        elif kind == 'maxpool3s2':
            bufs[op[2]] = maxpool3s2(bufs[op[1]])[0]
        elif kind == 'avgpool2':
            bufs[op[2]] = avgpool2(bufs[op[1]], q=q)[0]
        elif kind == 'gate':
            _, name, c, src, acc, accumulate = op
            bufs[acc] = gate(bufs[src], weights[name], bufs[acc] if accumulate else None, q=q)[0]
        elif kind == 'gate4':
            bufs[op[4]] = gate4([bufs[s_] for s_ in op[3]], weights[op[1]], q=q)[0]
        elif kind == 'add_relu':
            bufs[op[3]] = add_relu(bufs[op[1]], bufs[op[2]], q=q)[0]
        elif kind == 'gap':
            bufs[op[2]] = gap(bufs[op[1]])[0]
        elif kind == 'fc':
            _, name, cin, cout, src, dst = op
            out = bufs[dst] = fc(bufs[src], *weights[name])[0]
        else:
            raise NotImplementedError(kind)
    return out


def ulp16(v):
    """Spacing of fp16 numbers at |v| (float64)."""
    a = _d(v).abs().clamp_min(2.0 ** -14)
    return torch.exp2(torch.floor(torch.log2(a)) - 10)


def worst(got, want, bound):
    """(index tuple, error / bound) of the element with the largest ratio (0 / 0 counts as 0)."""
    err = (_d(got) - _d(want)).abs()
    ratio = torch.where(err == 0, torch.zeros_like(err), err / bound.clamp_min(1e-300))
    ratio = torch.where(torch.isnan(err), torch.full_like(err, math.inf), ratio)
    i = int(ratio.reshape(-1).argmax())
    idx = tuple(int(v) for v in torch.unravel_index(torch.tensor(i), ratio.shape))
    return idx, float(ratio.reshape(-1)[i])
