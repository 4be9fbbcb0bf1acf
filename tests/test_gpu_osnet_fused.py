"""GPU numerics of the fused OSNet kernels (csrc/osnet_fused.cu) against an fp32 PyTorch restatement of the same
layers (torchreid OSBlock: conv1 -> four Lite-3x3 streams), with fp16 rounding at the points where the kernels round
(x1, every pointwise output, every depthwise output).  Tolerance: the depthwise 3x3 accumulates its nine taps in
fp16 (HFMA2), so each level adds ~1e-3 relative noise on top of the storage rounding."""
import ctypes as C

import numpy as np
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu


def _h(t):
    return t.half().float()


def _streams_reference(x, w1, b1, pws, dws):
    """x: (n, h, w, cin) fp32 (already fp16-representable).  Returns 4 tails (n, h, w, mid) and their channel sums
    (the float64 reference of kernel S, oracle/nets64.py, with fp16 weights as the kernel reads them)."""
    from oracle import nets64
    tails = nets64.osb_streams(x, _h(w1), b1, [(_h(w), b) for w, b in pws], [(_h(w), b) for w, b in dws])
    tails = [t.float() for t, _ in tails]
    return tails, [t.sum((1, 2)) for t in tails]


def run_osb_streams(x, w1, b1, pws, dws):
    """x: (n, h, w, cin) fp16 cuda tensor; weights as fp32 numpy.  Returns (tails list, gap sums (n, 4, mid))."""
    from fastmot_b200 import _lib
    from fastmot_b200.devmem import stream_ptr
    from fastmot_b200.packing import pack_b_sw128
    lib = _lib.require_device()
    n, h, w, cin = x.shape
    mid = w1.shape[0]
    strips = lib.fm_osb_streams_strips(h, w, mid)
    assert strips > 0
    dev = x.device
    w1_d = torch.as_tensor(pack_b_sw128(w1)).to(dev)
    b1_d = torch.as_tensor(b1.astype(np.float32)).to(dev)
    pw_d = torch.as_tensor(np.concatenate([pack_b_sw128(wp) for wp, _ in pws])).to(dev)
    blobs = []
    for (wp, bp), (wd, bd) in zip(pws, dws):
        blobs.append(np.concatenate([wd.astype(np.float16).reshape(-1).view(np.uint8),
                                     bp.astype(np.float32).view(np.uint8), bd.astype(np.float32).view(np.uint8)]))
    dw_d = torch.as_tensor(np.concatenate(blobs)).to(dev)
    tails = [torch.full((n, mid // 8, h, w, 8), float('nan'), dtype=torch.float16, device=dev) for _ in range(4)]
    gap = torch.full((n, strips, 4, mid), float('nan'), dtype=torch.float32, device=dev)
    d = _lib.FmOsbStreams()
    d.x, d.n, d.h, d.w, d.cin, d.mid = x.data_ptr(), n, h, w, cin, mid
    d.w1, d.b1, d.pw, d.dw = w1_d.data_ptr(), b1_d.data_ptr(), pw_d.data_ptr(), dw_d.data_ptr()
    for i in range(4):
        d.tails[i] = tails[i].data_ptr()
    d.gap_part = gap.data_ptr()
    _lib.check(lib.fm_osb_streams(C.byref(d), stream_ptr()), "fm_osb_streams")
    torch.cuda.synchronize()
    # chunk-planar [n][mid / 8][h][w][8] -> NHWC
    tails = [t.permute(0, 2, 3, 1, 4).reshape(n, h, w, mid) for t in tails]
    return tails, gap.sum(1)


def _random_block(cin, mid, seed):
    rng = np.random.default_rng(seed)
    w1 = rng.normal(0, np.sqrt(2.0 / cin), (mid, cin)).astype(np.float32)
    b1 = rng.normal(0, 0.05, mid).astype(np.float32)
    pws = [(rng.normal(0, np.sqrt(1.0 / mid), (mid, mid)).astype(np.float32),
            rng.normal(0, 0.05, mid).astype(np.float32)) for _ in range(10)]
    dws = [(rng.normal(0, np.sqrt(2.0 / 9), (9, mid)).astype(np.float32),
            rng.normal(0, 0.05, mid).astype(np.float32)) for _ in range(10)]
    return w1, b1, pws, dws


@pytest.mark.parametrize("w,mid,h,cin,n", [(32, 64, 64, 64, 3), (32, 64, 64, 256, 2), (32, 64, 16, 64, 1),
                                           (16, 96, 32, 256, 3), (16, 96, 32, 384, 2),
                                           (8, 128, 16, 384, 5), (8, 128, 16, 512, 3)])
def test_osb_streams_vs_torch(w, mid, h, cin, n):
    w1, b1, pws, dws = _random_block(cin, mid, seed=w + cin)
    g = torch.Generator().manual_seed(cin + n)
    x = (torch.randn(n, h, w, cin, generator=g).abs() * 0.7).half()       # post-ReLU-like block input
    tails, gap = run_osb_streams(x.cuda(), w1, b1, pws, dws)
    t = lambda a: torch.as_tensor(a)
    want, want_gap = _streams_reference(x.float(), t(w1), t(b1), [(t(a), t(b)) for a, b in pws],
                                        [(t(a), t(b)) for a, b in dws])
    for s in range(4):
        got = tails[s].float().cpu()
        assert torch.isfinite(got).all(), s
        scale = float(want[s].abs().max()) + 1e-6
        err = float((got - want[s]).abs().max()) / scale
        assert err < 1.5e-2, (s, err)
        gerr = float((gap[:, s].cpu() - want_gap[s]).abs().max()) / (float(want_gap[s].abs().max()) + 1e-6)
        assert gerr < 5e-3, (s, gerr)


def test_osb_streams_border_rows_exact_zero_padding():
    """An all-zero input with zero biases except conv1's must give the same tails for every crop and respect the
    image border (the pointwise output is padded with zeros, not with its bias)."""
    w1, b1, pws, dws = _random_block(64, 64, seed=5)
    x = torch.zeros(2, 64, 32, 64, dtype=torch.float16)
    tails, _ = run_osb_streams(x.cuda(), w1, b1, pws, dws)
    t = lambda a: torch.as_tensor(a)
    want, _ = _streams_reference(x.float(), t(w1), t(b1), [(t(a), t(b)) for a, b in pws],
                                 [(t(a), t(b)) for a, b in dws])
    for s in range(4):
        got = tails[s].float().cpu()
        assert torch.equal(got[0], got[1])
        assert float((got - want[s]).abs().max()) / (float(want[s].abs().max()) + 1e-6) < 1.5e-2


@pytest.mark.parametrize("batch,graph", [(6, False), (200, True)])
def test_osnet_x1_fused_engine_vs_oracle_and_unfused(batch, graph, monkeypatch):
    """OSNet x1.0 with the fused OSBlock kernels == fp32 oracle (and == the layer-per-launch engine) at the batch the
    benchmark runs (200 crops, CUDA graph + PDL) and at a small eager batch."""
    from fastmot_b200.engine import OSNetEngine
    from oracle import nets
    g = torch.Generator().manual_seed(4)
    x = torch.randn(batch, 3, 256, 128, generator=g)
    inp = torch.zeros(batch, 256, 128, 8, dtype=torch.float16)
    inp[..., :3] = x.permute(0, 2, 3, 1).half()
    eng = OSNetEngine(1.0, max_batch=batch, use_graph=graph)
    assert eng.n_osb == 6
    eng.load_nhwc8(inp.cuda())
    got = eng.forward().clone()
    if graph:
        for _ in range(2):
            again = eng.forward()
        assert torch.equal(got, again)
    got = got.cpu()
    monkeypatch.setenv("FM_OSB_FUSED", "0")
    ref_eng = OSNetEngine(1.0, weights=eng.weights, max_batch=batch, use_graph=False)
    assert ref_eng.n_osb == 0
    ref_eng.load_nhwc8(inp.cuda())
    unfused = ref_eng.forward().cpu()
    assert float((got - unfused).abs().max()) < 5e-3, float((got - unfused).abs().max())
    nb = min(batch, 8)         # the CPU oracle is slow: first crops only
    want = nets.run_osnet(eng.ops, eng.weights, inp[:nb, ..., :3].float().permute(0, 3, 1, 2), nets.fp16_roundtrip)
    np.testing.assert_allclose(got.norm(dim=1).numpy(), 1.0, atol=1e-4)
    assert float((got[:nb] - want).abs().max()) < 5e-3, float((got[:nb] - want).abs().max())


def run_osb_merge(tails, gw, w3, b3, wd=None, bd=None, x=None, res=None):
    """tails: 4 x (n, h, w, mid) fp16 cuda (NHWC); returns out (n, h*w, cout) fp16."""
    from fastmot_b200 import _lib
    from fastmot_b200.devmem import stream_ptr
    from fastmot_b200.packing import pack_b_sw128
    lib = _lib.require_device()
    n, h, w, mid = tails[0].shape
    cout = w3.shape[0]
    ncta = lib.fm_osb_merge_ncta(mid, cout)
    assert ncta > 0
    dev = tails[0].device
    planar = [t.reshape(n, h, w, mid // 8, 8).permute(0, 3, 1, 2, 4).contiguous() for t in tails]
    strips = 2       # split the channel sums over two "strips" to exercise the strip reduction
    gap = torch.zeros(n, strips, 4, mid, dtype=torch.float32, device=dev)
    for s in range(4):
        tf = tails[s].float()
        gap[:, 0, s] = tf[:, :h // 2].sum((1, 2))
        gap[:, 1, s] = tf[:, h // 2:].sum((1, 2))
    wcat, bias = w3, b3.copy()
    if wd is not None:
        wcat = np.concatenate([wd, w3], 1)
        bias = bias + bd
    img = torch.as_tensor(np.concatenate([pack_b_sw128(wcat[r:r + ncta]) for r in range(0, cout, ncta)])).to(dev)
    bias_d = torch.as_tensor(bias.astype(np.float32)).to(dev)
    gws = [torch.as_tensor(np.ascontiguousarray(a, np.float32)).to(dev) for a in gw]
    out = torch.full((n, h * w, cout), float('nan'), dtype=torch.float16, device=dev)
    d = _lib.FmOsbMerge()
    d.n, d.hw, d.cout, d.mid, d.cr, d.strips = n, h * w, cout, mid, gw[0].shape[0], strips
    d.cin = wd.shape[1] if wd is not None else cout
    for i in range(4):
        d.tails[i] = planar[i].data_ptr()
    d.gap_part = gap.data_ptr()
    d.gw1, d.gb1, d.gw2, d.gb2 = (g.data_ptr() for g in gws)
    d.wimg, d.bias, d.out = img.data_ptr(), bias_d.data_ptr(), out.data_ptr()
    scratch = torch.zeros(4 * n * mid, dtype=torch.float32, device=dev)
    d.gate_scratch = scratch.data_ptr()
    d.x = x.data_ptr() if x is not None else None
    d.res = res.data_ptr() if res is not None else None
    _lib.check(lib.fm_osb_merge(C.byref(d), stream_ptr()), "fm_osb_merge")
    torch.cuda.synchronize()
    return out


@pytest.mark.parametrize("w,mid,h,cin,cout,n", [(32, 64, 64, 64, 256, 2), (32, 64, 64, 256, 256, 2),
                                                (16, 96, 32, 256, 384, 3), (16, 96, 32, 384, 384, 2),
                                                (8, 128, 16, 384, 512, 5), (8, 128, 16, 512, 512, 3)])
def test_osb_merge_vs_torch(w, mid, h, cin, cout, n):
    rng = np.random.default_rng(cin + cout)
    g = torch.Generator().manual_seed(cin)
    tails = [(torch.randn(n, h, w, mid, generator=g).abs() * 0.6).half() for _ in range(4)]
    cr = mid // 16
    gw = (rng.normal(0, np.sqrt(2.0 / mid), (cr, mid)), rng.normal(0, 0.1, cr),
          rng.normal(0, np.sqrt(2.0 / cr), (mid, cr)), rng.normal(0, 0.1, mid))
    w3 = rng.normal(0, np.sqrt(1.0 / mid), (cout, mid)).astype(np.float32)
    b3 = rng.normal(0, 0.05, cout).astype(np.float32)
    down = cin != cout
    if down:
        wd = rng.normal(0, np.sqrt(1.0 / cin), (cout, cin)).astype(np.float32)
        bd = rng.normal(0, 0.05, cout).astype(np.float32)
        x = (torch.randn(n, h * w, cin, generator=g).abs() * 0.7).half()
        got = run_osb_merge([t.cuda() for t in tails], gw, w3, b3, wd, bd, x=x.cuda())
    else:
        res = (torch.randn(n, h * w, cout, generator=g).abs() * 0.7).half()
        got = run_osb_merge([t.cuda() for t in tails], gw, w3, b3, res=res.cuda())
    from oracle import nets64
    t = lambda a: torch.as_tensor(np.asarray(a, np.float32))
    gap = torch.stack([torch.stack([tl.float()[:, :h // 2].sum((1, 2)), tl.float()[:, h // 2:].sum((1, 2))], 1)
                       for tl in tails], 2)                        # the strip sums run_osb_merge hands the kernel
    gwt = tuple(t(a) for a in gw)
    if down:
        want, _ = nets64.osb_merge(tails, gap, gwt, _h(t(w3)), t(t(b3) + t(bd)), x=x.reshape(n, h, w, cin),
                                   wd=_h(t(wd)))
    else:
        want, _ = nets64.osb_merge(tails, gap, gwt, _h(t(w3)), t(b3), res=res.reshape(n, h, w, cout))
    want = want.float().reshape(n, h * w, cout)
    gotc = got.float().cpu()
    assert torch.isfinite(gotc).all()
    err = float((gotc - want).abs().max()) / (float(want.abs().max()) + 1e-6)
    assert err < 4e-3, err


@pytest.mark.parametrize("n", [1, 5])
def test_osnet_stem_vs_torch(n):
    """Fused 7x7/2 conv + ReLU + 3x3/2 max-pool (TMA 5-D window tiles) against fp32 torch."""
    from fastmot_b200 import _lib
    from fastmot_b200.devmem import ptr, stream_ptr
    from fastmot_b200.packing import pack_b_sw64
    lib = _lib.require_device()
    rng = np.random.default_rng(7)
    w7 = rng.normal(0, np.sqrt(2.0 / 147), (64, 7, 7, 3)).astype(np.float32)
    b7 = rng.normal(0, 0.05, 64).astype(np.float32)
    g = torch.Generator().manual_seed(n)
    x = torch.randn(n, 256, 128, 3, generator=g).half()
    xin = torch.zeros(n, 264, 136, 4, dtype=torch.float16)
    xin[:, 4:-4, 4:-4, :3] = x
    wk = np.zeros((64, 7, 8, 4), np.float32)
    wk[:, :, 1:8, :3] = w7
    img = torch.as_tensor(pack_b_sw64(wk.reshape(64, 224))).cuda()
    out = torch.full((n, 64, 32, 64), float('nan'), dtype=torch.float16, device="cuda")
    xin_d, b_d = xin.cuda(), torch.as_tensor(b7).cuda()
    _lib.check(lib.fm_osnet_stem(ptr(xin_d), n, ptr(img), ptr(b_d), ptr(out), stream_ptr()), "fm_osnet_stem")
    torch.cuda.synchronize()
    wt = _h(torch.as_tensor(w7)).permute(0, 3, 1, 2).contiguous()
    y = F.relu(F.conv2d(x.float().permute(0, 3, 1, 2), wt, torch.as_tensor(b7), stride=2, padding=3))
    want = F.max_pool2d(_h(y), 3, 2, 1).permute(0, 2, 3, 1)
    got = out.float().cpu()
    assert torch.isfinite(got).all()
    err = float((got - want).abs().max()) / (float(want.abs().max()) + 1e-6)
    assert err < 3e-3, err


@pytest.mark.parametrize("n,cin,cout,relu", [(200, 512, 512, 0), (37, 512, 512, 1), (16, 256, 128, 0), (6, 512, 512, 0)])
def test_fc_norm_vs_torch(n, cin, cout, relu):
    """ReID head: fc + L2 normalisation (feature_extractor.py:62-74): cluster kernel (n >= 16) and the small-batch kernel."""
    import torch.nn.functional as F
    from fastmot_b200 import _lib
    from fastmot_b200.devmem import ptr, stream_ptr
    lib = _lib.require_device()
    g = torch.Generator().manual_seed(n)
    x = torch.randn(n, cin, generator=g)
    w = torch.randn(cout, cin, generator=g) * 0.05
    b = torch.randn(cout, generator=g) * 0.1
    xd, wd, bd = x.cuda(), w.cuda(), b.cuda()
    out = torch.zeros(n, cout, dtype=torch.float32, device="cuda")
    _lib.check(lib.fm_fc_norm(ptr(xd), ptr(wd), ptr(bd), ptr(out), n, cin, cout, relu, 1, stream_ptr()), "fm_fc_norm")
    torch.cuda.synchronize()
    y = x @ w.t() + b
    if relu:
        y = y.clamp_min(0)
    want = F.normalize(y, dim=1)
    assert float((out.cpu() - want).abs().max()) < 2e-5
    out2 = torch.zeros_like(out)
    _lib.check(lib.fm_fc_norm(ptr(xd), ptr(wd), ptr(bd), ptr(out2), n, cin, cout, relu, 1, stream_ptr()), "fm_fc_norm")
    torch.cuda.synchronize()
    assert torch.equal(out, out2)          # deterministic (fixed summation order across the cluster)
