"""Every launch of the ReID engine, one at a time, against the float64 reference of what it computes (oracle/nets64.py),
at the batch sizes the product runs.

For each recorded launch (OSNetEngine.trace describes it) the test
  1. checks that every view it reads still holds, bit for bit, what its producer wrote (buffer recycling must not
     overwrite a live tensor),
  2. runs it alone on the stream the replay uses,
  3. compares every output element of every crop with the float64 reference computed from the inputs as the kernel
     read them (teacher forcing), within the per-element bound of the kernel's rounding model.
A failure names the launch, the op kind, the crop / y / x / channel of the worst element and its error / bound.
The largest error / bound per kind is printed (pytest -s) so the headroom is visible."""
import time

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

CHUNK = 50          # crops per float64 reference evaluation (bounds the device memory of the stage-1 chain)


def _nhwc(v, a):
    """A view's array as the reference sees it: NHWC for activations, as stored otherwise."""
    return a.permute(0, 2, 3, 1, 4).reshape(a.shape[0], v.h, v.w, v.c) if v.layout == 'planar8' else a


def _bits(t):
    t = t.contiguous()
    return t.view(torch.int16) if t.dtype == torch.float16 else t.view(torch.int32)


def _dw_model(h, w, c):
    """Which fm_dwconv3 kernel runs (nn_vec.cu fm_vec_dwconv3): the tiled HFMA2 one or an fp32 one."""
    if c % 8 == 0 and w % 4 == 0 and h >= 8 and ((8 + 2) * w + 9) * c * 2 <= 96 * 1024:
        return 'rows3'
    return 'fp32'


def _h(a, dev):
    """Host fp32 weights as the kernels read them after the fp16 conversion (packing.py, engine.py)."""
    return torch.as_tensor(np.asarray(a, np.float32)).to(dev).half().double()


def _f(a, dev):
    return torch.as_tensor(np.asarray(a, np.float32)).to(dev).double()


def _reference(eng, e, ins):
    """(want, bound) per output view of trace entry e; ins: its input arrays (float64, NHWC / as stored)."""
    from oracle import nets64 as R
    ops, W, P, dev = eng.ops, eng.weights, eng._params, ins[0].device
    op = ops[e.ops[0]]
    k = e.kind
    if k == 'stem':
        return [R.stem(ins[0], _h(W[op[1]][0], dev), _f(W[op[1]][1], dev))]
    if k in ('conv', 'conv+add'):
        _, name, cin, cout, ks, stride, pad, act, src, dst = op
        wd, bd = P[name]
        if k == 'conv':
            return [R.conv(ins[0], wd, bd, stride, pad, act)]
        return [R.conv(ins[0], wd, bd, stride, pad, 'relu', res=ins[1], res_first=True)]
    if k == 'dw':
        wd, bd = P[op[1]]
        _, h, w, c = ins[0].shape
        return [R.dw(ins[0], wd, bd, op[3], _dw_model(h, w, c))]
    if k == 'maxpool3s2':
        return [R.maxpool3s2(ins[0])]
    if k == 'avgpool2':
        return [R.avgpool2(ins[0])]
    if k == 'gate':
        return [R.gate(ins[0], P[op[1]], ins[1] if op[5] else None)]
    if k == 'gate4':
        return [R.gate4(ins[:4], P[op[1]])]
    if k == 'gate4_pooled':
        return [R.gate4_pooled(ins[:4], ins[4], P[op[1]])]
    if k == 'add_relu':
        return [R.add_relu(ins[0], ins[1])]
    if k == 'gap':
        return [R.gap(ins[0])]
    if k == 'fc':
        return [R.fc(ins[0], *P[op[1]])]
    if k == 'S':
        mid, cin = op[3], op[2]
        w1 = _h(W[op[1]][0], dev).reshape(mid, cin)
        pws, dws = [], []
        for i in range(10):
            pw, dwo = ops[e.ops[0] + 1 + 2 * i], ops[e.ops[0] + 2 + 2 * i]
            pws.append((_h(W[pw[1]][0], dev).reshape(mid, mid), _f(W[pw[1]][1], dev)))
            dws.append((_h(W[dwo[1]][0], dev), _f(W[dwo[1]][1], dev)))
        return R.osb_streams(ins[0], w1, _f(W[op[1]][1], dev), pws, dws)
    if k == 'G':
        seq = [ops[i] for i in e.ops]
        c3 = [o for o in seq if o[0] == 'conv' and o[8] == op[4]][0]
        ds = [o for o in seq if o[0] == 'conv' and o is not c3]
        cout, mid = c3[3], c3[2]
        w3 = _h(W[c3[1]][0], dev).reshape(cout, mid)
        bias = np.asarray(W[c3[1]][1], np.float32).copy()
        if ds:
            bias += np.asarray(W[ds[0][1]][1], np.float32)
            wdn = _h(W[ds[0][1]][0], dev).reshape(cout, ds[0][2])
            return [R.osb_merge(ins[:4], ins[4], P[op[1]], w3, _f(bias, dev), x=ins[5], wd=wdn)]
        return [R.osb_merge(ins[:4], ins[4], P[op[1]], w3, _f(bias, dev), res=ins[5])]
    raise NotImplementedError(k)


def run_launch_by_launch(eng, crops, label):
    """Runs eng's launches one by one on crops (B, 256, 128, 8) fp16 and checks them; returns {kind: worst ratio}."""
    from fastmot_b200.devmem import stream_ptr
    from oracle import nets64 as R
    n = eng.max_batch
    assert len(eng.trace) == len(eng.launches)
    assert not eng._live, f"buffers still held after their last reader: {sorted(eng._live)}"
    eng.load_nhwc8(crops)
    last_read = {}
    for i, e in enumerate(eng.trace):
        for v in e.ins:
            last_read[v.name] = i
    first = eng.trace[0].ins[0]
    snap = {first.name: first.array(n).clone()}
    worst = {}
    sp = stream_ptr()
    torch.cuda.synchronize()
    for i, e in enumerate(eng.trace):
        where = f"{label}: launch {i} ({e.kind}, ops {e.ops[0]}..{e.ops[-1]})"
        for v in e.ins:                                            # 1. lifetime
            assert v.name in snap, (where, v.name, "read before it was written")
            assert torch.equal(_bits(v.array(n)), _bits(snap[v.name])), \
                (where, f"input '{v.name}' was overwritten after its producer wrote it")
        ins = [_nhwc(v, v.array(n).double()) for v in e.ins]
        eng.launches[i](sp)                                        # 2. the launch alone
        torch.cuda.synchronize()
        outs = [v.array(n).clone() for v in e.outs]
        for v, o in zip(e.outs, outs):
            snap[v.name] = o
        for nm in [nm for nm, j in last_read.items() if j == i]:
            snap.pop(nm, None)
        got = [_nhwc(v, o.double()) for v, o in zip(e.outs, outs)]
        ratio = 0.0
        for c0 in range(0, n, CHUNK):                              # 3. values, every crop
            sl = slice(c0, min(n, c0 + CHUNK))
            refs = _reference(eng, e, [a[sl] for a in ins])
            if e.kind == 'S':                                      # strip sums of the tails the kernel stored
                refs.append(R.strip_sums([g[sl] for g in got[:4]], e.outs[4].strips))
            assert len(refs) == len(got), where
            for j, ((want, bound), g) in enumerate(zip(refs, got)):
                g = g[sl]
                assert g.shape == want.shape, (where, j, tuple(g.shape), tuple(want.shape))
                idx, r = R.worst(g, want, bound)
                if r > 1.0:
                    pos = (c0 + idx[0],) + idx[1:]
                    pytest.fail(f"{where}: output '{e.outs[j].name}' ({e.outs[j].layout}) at crop/y/x/ch {pos}: "
                                f"got {float(g[idx]):.6g}, want {float(want[idx]):.6g}, bound {float(bound[idx]):.3g}, "
                                f"error/bound {r:.3g}")
                ratio = max(ratio, r)
        worst[e.kind] = max(worst.get(e.kind, 0.0), ratio)
    return worst


def _crops(n, seed, hw=(256, 128)):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(n, 3, hw[0], hw[1], generator=g)
    inp = torch.zeros(n, hw[0], hw[1], 8, dtype=torch.float16)
    inp[..., :3] = x.permute(0, 2, 3, 1).half()
    return inp.cuda()


def _report(label, worst, t0):
    print(f"\n[osnet ops] {label}: {time.time() - t0:.1f} s; max error/bound per kind: " +
          ", ".join(f"{k} {v:.3f}" for k, v in sorted(worst.items())))


@pytest.mark.parametrize("batch", [200, 13])
def test_osnet_x1_fused_launch_by_launch(batch):
    """Config 3 (200 crops: the 4-CTA clusters of kernel S run in several waves) and a batch that is not a multiple
    of 8."""
    from fastmot_b200.engine import OSNetEngine
    t0 = time.time()
    eng = OSNetEngine(1.0, max_batch=batch, use_graph=False)
    assert eng.n_osb == 6 and eng.fuse_stem
    kinds = {e.kind for e in eng.trace}
    assert {'stem', 'S', 'G', 'conv', 'avgpool2', 'gap', 'fc'} <= kinds, kinds
    worst = run_launch_by_launch(eng, _crops(batch, 100 + batch), f"x1.0 fused, batch {batch}")
    _report(f"x1.0 fused, batch {batch}", worst, t0)


def test_osnet_x1_per_layer_launch_by_launch(monkeypatch):
    """The per-layer path (FM_OSB_FUSED=0): pointwise convs at mid 64 / 96 / 128, depthwise, gate4, and conv3 with
    the residual + ReLU in the conv_tc epilogue (FM_ACT_AFTER_RESIDUAL)."""
    from fastmot_b200.engine import OSNetEngine
    monkeypatch.setenv("FM_OSB_FUSED", "0")
    t0 = time.time()
    eng = OSNetEngine(1.0, max_batch=24, use_graph=False)
    assert eng.n_osb == 0
    kinds = [e.kind for e in eng.trace]
    assert kinds.count('conv+add') == 6 and 'gate4' in kinds and 'maxpool3s2' in kinds
    mids = {eng.ops[e.ops[0]][2] for e in eng.trace if e.kind == 'dw'}
    assert mids == {64, 96, 128}, mids
    worst = run_launch_by_launch(eng, _crops(24, 7), "x1.0 per layer, batch 24")
    _report("x1.0 per layer, batch 24", worst, t0)


def test_osnet_x025_launch_by_launch():
    """Config 2: OSNet x0.25 at the 56-crop bucket, the whole per-layer path (SIMT 1x1 convs at 16 / 24 channels,
    conv_tc, depthwise, max / avg pool, gate4, add)."""
    from fastmot_b200.engine import OSNetEngine
    t0 = time.time()
    eng = OSNetEngine(0.25, max_batch=56, use_graph=False)
    assert eng.n_osb == 0 and eng.n_simt > 0
    worst = run_launch_by_launch(eng, _crops(56, 25), "x0.25, batch 56")
    _report("x0.25, batch 56", worst, t0)


@pytest.mark.parametrize("ch", [64, 10])
def test_custom_backbone_launch_by_launch(ch):
    """The imported non-OSNet graph of test_onnx_import (two-stream 'gate' accumulate, plain residual add, 3x3 stem
    through the SIMT conv).  10 channels reach the scalar (non-16-byte) kernels of max-pool, depthwise, channel gate,
    2x2 average pool (20 channels) and global average pool."""
    from test_onnx_import import _custom_graph
    from fastmot_b200.engine import OSNetEngine
    from fastmot_b200.models import onnx_io
    from fastmot_b200.models.onnx_import import import_reid_onnx
    ops, w, in_shape, dim = import_reid_onnx(onnx_io.serialize(_custom_graph(ch)))
    t0 = time.time()
    eng = OSNetEngine(None, weights=w, input_hw=in_shape[1:], feature_dim=dim, max_batch=24, use_graph=False, ops=ops)
    kinds = [e.kind for e in eng.trace]
    assert kinds.count('gate') == 2 and 'add_relu' in kinds and 'dw' in kinds, kinds
    worst = run_launch_by_launch(eng, _crops(24, 3, tuple(in_shape[1:])), f"custom {ch} ch, batch 24")
    _report(f"custom {ch} ch, batch 24", worst, t0)
