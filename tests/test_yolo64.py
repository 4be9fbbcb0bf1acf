"""CPU checks of the float64 Darknet reference (oracle/nets64.py): composed over whole detectors it computes what the
fp32 oracle computes, and its error bounds admit a result rounded the way the kernels round but reject the faults a
wrong detector kernel would make."""
import numpy as np
import pytest
import torch

from fastmot_b200.models import darknet
from oracle import detect, nets, nets64 as R

ACTS = ['linear', 'leaky', 'relu', 'logistic', 'swish', 'mish']


@pytest.mark.parametrize("name", ['yolov4-tiny', 'yolov4-csp', 'yolov4-p5'])
def test_float64_darknet_executor_matches_oracle(name):
    """Same layer semantics as oracle.nets.run_darknet (routes, group splits, SPP pools, shortcuts, upsampling), both
    evaluated in float64 so that the deep nets' amplification of fp32 rounding does not hide a difference."""
    layers = darknet.BUILDERS[name]()
    w = darknet.synthetic_weights(layers, 3, head_obj_bias=-3.0)
    w64 = {i: (a.astype(np.float64), b.astype(np.float64)) for i, (a, b) in w.items()}
    x = torch.rand(1, 3, 96, 64, generator=torch.Generator().manual_seed(0), dtype=torch.float64)
    got = R.run_darknet64(layers, w, x)
    want = nets.run_darknet(layers, w64, x)
    assert len(got) == len(want) >= 2
    for g, h in zip(got, want):
        assert g.shape == h.shape
        assert float((g - h).abs().max() / h.abs().max()) < 1e-5


def _passes(got, want, bound):
    return R.worst(got, want, bound)[1] <= 1.0


def _ulp_noise(want, seed):
    """want moved by one fp16 ulp at a random two thirds of the elements: what a kernel that rounds its fp32 result to
    the other neighbour of the same exact value stores."""
    g = torch.Generator().manual_seed(seed)
    sign = torch.randint(0, 3, want.shape, generator=g).double() - 1
    return R.f16(want + sign * R.ulp16(want))


def _h(shape, scale, g):
    return (torch.randn(*shape, generator=g) * scale).half().double()


def _conv_case(g, h=13, w=13, cin=512, cout=64, k=3):
    x = _h((1, h, w, cin), 1.0, g)
    wt = _h((cout, k, k, cin), (2.0 / (k * k * cin)) ** 0.5, g)
    b = (torch.randn(cout, generator=g) * 0.3).float().double()
    return x, wt, b


@pytest.mark.parametrize("act", ACTS)
def test_conv_bound_admits_one_ulp_for_every_activation(act):
    g = torch.Generator().manual_seed(ACTS.index(act))
    x, wt, b = _conv_case(g, cin=128)
    want, bound = R.conv(x, wt, b, 1, 1, act)
    assert _passes(_ulp_noise(want, 1), want, bound)
    res = _h((1, 13, 13, 64), 1.0, g)
    want, bound = R.conv(x, wt, b, 1, 1, act, res=res, res_first=False)         # the fused Darknet shortcut
    assert _passes(_ulp_noise(want, 2), want, bound)
    assert not _passes(R.conv(x, wt, b, 1, 1, act, res=res, res_first=True)[0], want, bound) or act == 'linear'
    # the shortcut add is exact up to one fp32 rounding, so only the fp16 neighbour a value within u32 of a rounding
    # boundary may take is admitted, not an arbitrary ulp
    want, bound = R.add_act(x, x.flip(1), act)
    exact = R.add_act(x, x.flip(1), act, q=False)[0]
    for sign in (1, -1):
        assert _passes(R.f16(exact * (1 + sign * R.U32)), want, bound)
    if act in ('linear', 'relu'):
        assert not _passes(_ulp_noise(want, 3), want, bound)


def test_conv_bounds_reject_concat_shift_stale_tile_and_dropped_k_slice():
    g = torch.Generator().manual_seed(11)
    x, wt, b = _conv_case(g, cin=512, cout=64)
    want, bound = R.conv(x, wt, b, 1, 1, 'leaky')
    assert _passes(_ulp_noise(want, 4), want, bound)
    bad = want.clone()                                       # the write landed 8 channels off in the concat buffer
    bad[..., 8:] = want[..., :-8]
    assert not _passes(bad, want, bound)
    # the ragged last tile of the 13 x 13 plane (pixels 128 .. 168) left as a previous frame wrote it
    other = R.conv(_h((1, 13, 13, 512), 1.0, g), wt, b, 1, 1, 'leaky')[0]
    bad = want.clone().reshape(-1, 64)
    bad[128:] = other.reshape(-1, 64)[128:]
    assert not _passes(bad.reshape(want.shape), want, bound)
    wt2 = wt.clone()                                         # K slice 64 .. 127 of every tap dropped
    wt2[..., 64:128] = 0
    assert not _passes(R.conv(x, wt2, b, 1, 1, 'leaky')[0], want, bound)


def test_mish_bound_rejects_leaky_in_one_channel_group():
    g = torch.Generator().manual_seed(12)
    x, wt, b = _conv_case(g, cin=256, cout=64, k=1)
    want, bound = R.conv(x, wt, b, 1, 0, 'mish')
    assert _passes(_ulp_noise(want, 5), want, bound)
    bad = want.clone()
    bad[..., 8:16] = R.conv(x, wt, b, 1, 0, 'leaky')[0][..., 8:16]
    assert not _passes(bad, want, bound)


def test_pool_upsample_and_copy_are_exact():
    g = torch.Generator().manual_seed(13)
    x = _h((1, 20, 20, 32), 1.0, g)
    want, bound = R.maxpool(x, 9, 1)
    assert float(bound.abs().max()) == 0.0 and want.shape == x.shape
    # the declared window and source of the SPP pools: 9 = 5 o 5, 13 = 5 o 9
    p5 = R.maxpool(x, 5, 1)[0]
    assert torch.equal(R.maxpool(p5, 5, 1)[0], want)
    assert torch.equal(R.maxpool(want, 5, 1)[0], R.maxpool(x, 13, 1)[0])
    assert not _passes(p5, want, bound)                      # SPP 9 computed as 5
    # same-upper padding of an even window on an odd plane (tiny's 2 x 2 / 2 pools) matches the fp32 oracle
    xo = x[:, :13, :13]
    want = R.maxpool(xo, 2, 2)[0]
    assert torch.equal(want, nets._same_upper_pool(xo.permute(0, 3, 1, 2), 2, 2).permute(0, 2, 3, 1))
    up, ub = R.upsample(x, 2)
    assert up.shape == (1, 40, 40, 32) and float(ub.abs().max()) == 0.0
    assert not _passes(torch.roll(up, 1, 1), up, ub)         # one row off
    cp, cb = R.copy(x)
    assert torch.equal(cp, x) and float(cb.abs().max()) == 0.0


def _head(g, A, nc, H, W, new_coords):
    t = torch.randn(A, 5 + nc, H, W, generator=g)
    if new_coords:
        t = torch.sigmoid(t * 1.5)
    else:
        t[:, 4] += 1.0
    return t.reshape(A * (5 + nc), H, W).half().double()


@pytest.mark.parametrize("name", ['YOLOv4Tiny', 'YOLOv4', 'YOLOv4CSP', 'YOLOv4P5'])
def test_decode64_matches_oracle_decode(name):
    """decode64 is yolo_decode (then the detector's scaling to pixels): bit for bit for new coords, within its bound
    (which the fp32 numpy oracle, with its own exp, meets) for old coords."""
    from fastmot_b200 import models
    m = models.YOLO.get_model(name)
    g = torch.Generator().manual_seed(14)
    _, H, W = m.INPUT_SHAPE
    size, off = (1920.0, 1920.0), (0.0, 420.0)
    for f, anchors, scale in zip(m.LAYER_FACTORS, m.ANCHORS, m.SCALES):
        head = _head(g, len(anchors) // 2, m.NUM_CLASSES, H // f, W // f, m.NEW_COORDS)
        want, bound = R.decode64(head, anchors, scale, (W, H), m.NUM_CLASSES, m.NEW_COORDS, size, off)
        d = detect.yolo_decode(head.float().numpy(), anchors, scale, (W, H), m.NUM_CLASSES, m.NEW_COORDS)
        px = d[:, :4].astype(np.float64) * np.array(size * 2)
        d[:, :4] = px.astype(np.float32)
        d[:, :2] = (d[:, :2].astype(np.float64) - np.array(off)).astype(np.float32)
        ref = torch.as_tensor(d).double()
        assert torch.equal(ref[:, 5], want[:, 5])
        err = (ref - want[:, :7]).abs()
        if m.NEW_COORDS:
            assert float(err.max()) == 0.0
        else:
            assert bool((err <= bound[:, :7]).all()), float((err / bound[:, :7].clamp_min(1e-300)).max())
            assert bool((bound[:, :4] <= 1e-5 * want[:, :4].abs() + 0.01).all())     # far below a pixel


@pytest.mark.parametrize("name", ['YOLOv4Tiny', 'YOLOv4CSP'])
def test_decode64_rejects_swapped_head_anchors(name):
    from fastmot_b200 import models
    m = models.YOLO.get_model(name)
    g = torch.Generator().manual_seed(15)
    _, H, W = m.INPUT_SHAPE
    f = m.LAYER_FACTORS[0]
    head = _head(g, len(m.ANCHORS[0]) // 2, m.NUM_CLASSES, H // f, W // f, m.NEW_COORDS)
    want, bound = R.decode64(head, m.ANCHORS[0], m.SCALES[0], (W, H), m.NUM_CLASSES, m.NEW_COORDS)
    assert _passes(want + 0.5 * bound, want, bound)
    bad = R.decode64(head, m.ANCHORS[1], m.SCALES[0], (W, H), m.NUM_CLASSES, m.NEW_COORDS)[0]
    assert not _passes(bad, want, bound)
