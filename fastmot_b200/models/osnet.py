"""OSNet (Zhou et al., ICCV'19; torchreid `osnet_x1_0` / `osnet_x0_25`) as an op list for the ReID engine.

The reference only ships descriptors (fastmot/models/reid.py:95-109: input 3x256x128, 512-d output) and downloads
the ONNX files; the architecture below restates the published network (SURVEY.md Appendix D): 7x7/2 stem + 3x3/2
maxpool, three stages of two OSBlocks (1x1 reduce -> four streams of 1..4 "Lite 3x3" = 1x1 linear + depthwise 3x3
+ BN + ReLU -> shared channel gate -> sum -> 1x1 expand + residual), 1x1 + 2x2 avg-pool transitions after stages
1 and 2, 1x1 conv, global average pool, FC 512 + BN + ReLU.  All BNs are folded into the preceding conv.

Op tuples (executed by fastmot_b200.engine.OSNetEngine and, in fp32 torch, by oracle/nets.py):
  ('conv', name, cin, cout, k, stride, pad, act, src, dst)      dense conv, weights[name] = (w[out][kh][kw][in], b)
  ('dw',   name, c, act, src, dst)                              depthwise 3x3 s1 p1, weights[name] = (w[9][c], b)
  ('maxpool3s2', src, dst) / ('avgpool2', src, dst)
  ('gate', name, c, src, acc, accumulate)                       acc (+)= src * sigmoid(fc2(relu(fc1(gap(src)))))
  ('gate4', name, c, (s0, s1, s2, s3), acc)                    acc = sum_i s_i * gate(s_i), shared gate weights
  ('add_relu', a, b, dst)
  ('gap', src, dst) / ('fc', name, cin, cout, src, dst)
`src`/`dst` are symbolic buffer names.
"""
import numpy as np


def build_osnet(width=1.0, feature_dim=512):
    ch = [int(64 * width), int(256 * width), int(384 * width), int(512 * width)]
    ops = []
    ops.append(('conv', 'conv1', 3, ch[0], 7, 2, 3, 'relu', 'input', 'x'))
    ops.append(('maxpool3s2', 'x', 'x'))
    cur = 'x'
    uid = [0]

    def buf(prefix):
        uid[0] += 1
        return f'{prefix}{uid[0]}'

    def osblock(name, cin, cout, src):
        mid = cout // 4
        x1 = buf('t')
        ops.append(('conv', f'{name}.conv1', cin, mid, 1, 1, 0, 'relu', src, x1))
        acc = buf('t')
        tails = []
        for s in range(4):
            prev = x1
            for j in range(s + 1):
                a, b2 = buf('t'), buf('t')
                ops.append(('conv', f'{name}.conv2{"abcd"[s]}.{j}.pw', mid, mid, 1, 1, 0, 'linear', prev, a))
                ops.append(('dw', f'{name}.conv2{"abcd"[s]}.{j}.dw', mid, 'relu', a, b2))
                prev = b2
            tails.append(prev)
        # the four streams share one gate module; acc = sum_s gate(x_s) * x_s in a single pass
        ops.append(('gate4', f'{name}.gate', mid, tuple(tails), acc))
        ident = src
        if cin != cout:
            ident = buf('t')
            ops.append(('conv', f'{name}.downsample', cin, cout, 1, 1, 0, 'linear', src, ident))
        x3 = buf('t')
        ops.append(('conv', f'{name}.conv3', mid, cout, 1, 1, 0, 'linear', acc, x3))
        out = buf('t')
        ops.append(('add_relu', x3, ident, out))      # the engine fuses this into conv3's epilogue
        return out

    for stage in range(3):
        cin, cout = ch[stage], ch[stage + 1]
        cur = osblock(f'conv{stage + 2}.0', cin, cout, cur)
        cur = osblock(f'conv{stage + 2}.1', cout, cout, cur)
        if stage < 2:
            t = buf('t')
            ops.append(('conv', f'conv{stage + 2}.trans', cout, cout, 1, 1, 0, 'relu', cur, t))
            t2 = buf('t')
            ops.append(('avgpool2', t, t2))
            cur = t2
    t = buf('t')
    ops.append(('conv', 'conv5', ch[3], ch[3], 1, 1, 0, 'relu', cur, t))
    ops.append(('gap', t, 'pooled'))
    ops.append(('fc', 'fc', ch[3], feature_dim, 'pooled', 'feat'))
    return ops


def synthetic_weights(ops, seed_base=5000, reduction=16, calibrate=True):
    """Seeded He-normal weights with folded BN for every parametrised op."""
    w = {}
    k = 0
    for op in ops:
        kind = op[0]
        if kind == 'conv':
            _, name, cin, cout, ks = op[:5]
            rng = np.random.default_rng(seed_base + k)
            w[name] = (rng.normal(0, np.sqrt(2.0 / (ks * ks * cin)), (cout, ks, ks, cin)).astype(np.float32),
                       rng.normal(0, 0.02, cout).astype(np.float32))
        elif kind == 'dw':
            _, name, c = op[:3]
            rng = np.random.default_rng(seed_base + k)
            w[name] = (rng.normal(0, np.sqrt(2.0 / 9), (9, c)).astype(np.float32),
                       rng.normal(0, 0.02, c).astype(np.float32))
        elif kind in ('gate', 'gate4'):
            _, name, c = op[:3]
            if name not in w:
                rng = np.random.default_rng(seed_base + k)
                cr = max(c // reduction, 1)
                w[name] = (rng.normal(0, np.sqrt(2.0 / c), (cr, c)).astype(np.float32),
                           rng.normal(0, 0.02, cr).astype(np.float32),
                           rng.normal(0, np.sqrt(2.0 / cr), (c, cr)).astype(np.float32),
                           rng.normal(0, 0.02, c).astype(np.float32))
        elif kind == 'fc':
            _, name, cin, cout = op[:4]
            rng = np.random.default_rng(seed_base + k)
            w[name] = (rng.normal(0, np.sqrt(2.0 / cin), (cout, cin)).astype(np.float32),
                       rng.normal(0.0, 0.02, cout).astype(np.float32))
        k += 1
    if calibrate:
        from .calibrate import calibrate_osnet
        w = calibrate_osnet(ops, w)
    return w


def infer_shapes(ops, h=256, w=128):
    """The (c, h, w) of the tensor each op writes, in op order, for a 3-channel h x w input.  A list per op, not a
    dict per name: an op list may bind a name twice (the stem writes 'x' with the conv and again with the pool)."""
    named = {'input': (3, h, w)}
    shapes = []
    for op in ops:
        kind = op[0]
        if kind == 'conv':
            _, _, _, cout, ks, stride, pad, _, src, dst = op
            _, hh, ww = named[src]
            shape = (cout, (hh + 2 * pad - ks) // stride + 1, (ww + 2 * pad - ks) // stride + 1)
        elif kind == 'dw':
            shape, dst = (op[2],) + named[op[4]][1:], op[5]
        elif kind == 'maxpool3s2':
            c, hh, ww = named[op[1]]
            shape, dst = (c, (hh + 2 - 3) // 2 + 1, (ww + 2 - 3) // 2 + 1), op[2]
        elif kind == 'avgpool2':
            c, hh, ww = named[op[1]]
            shape, dst = (c, hh // 2, ww // 2), op[2]
        elif kind == 'gate':
            shape, dst = (op[2],) + named[op[3]][1:], op[4]
        elif kind == 'gate4':
            shape, dst = (op[2],) + named[op[3][0]][1:], op[4]
        elif kind == 'add_relu':
            shape, dst = named[op[1]], op[3]
        elif kind == 'gap':
            shape, dst = (named[op[1]][0], 1, 1), op[2]
        elif kind == 'fc':
            shape, dst = (op[3], 1, 1), op[5]
        else:
            raise NotImplementedError(kind)
        named[dst] = shape
        shapes.append(shape)
    return shapes


def count_macs(ops, h=256, w=128):
    """Multiply-accumulates per crop (dense convs + depthwise + fc)."""
    total = 0
    for op, (c, ho, wo) in zip(ops, infer_shapes(ops, h, w)):
        if op[0] == 'conv':
            total += op[2] * c * op[4] * op[4] * ho * wo
        elif op[0] == 'dw':
            total += 9 * c * ho * wo
        elif op[0] == 'fc':
            total += op[2] * op[3]
    return total
