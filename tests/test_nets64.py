"""CPU checks of the float64 reference (oracle/nets64.py): composed over whole networks it is the fp32 oracle, and its
error bounds admit a result rounded the way the kernels round but reject the faults a wrong kernel would make."""
import pytest
import torch

from fastmot_b200.models import osnet
from oracle import nets, nets64 as R


def _x(n, hw=(256, 128), seed=0):
    return torch.randn(n, 3, hw[0], hw[1], generator=torch.Generator().manual_seed(seed))


@pytest.mark.parametrize("width", [1.0, 0.25])
def test_float64_executor_matches_fp32_oracle(width):
    ops = osnet.build_osnet(width)
    w = osnet.synthetic_weights(ops)
    x = _x(2)
    got = R.run_ops(ops, w, x)
    want = nets.run_osnet(ops, w, x).double()
    assert float((got - want).abs().max()) < 1e-5


def test_float64_executor_matches_fp32_oracle_custom_graph():
    from test_onnx_import import _custom_graph
    from fastmot_b200.models import onnx_io
    from fastmot_b200.models.onnx_import import import_reid_onnx
    ops, w, in_shape, dim = import_reid_onnx(onnx_io.serialize(_custom_graph(16)))
    x = _x(3, in_shape[1:], seed=1)
    got = R.run_ops(ops, w, x)
    want = nets.run_osnet(ops, w, x).double()
    assert got.shape == (3, dim)
    assert float((got - want).abs().max()) < 1e-5


def _passes(got, want, bound):
    return R.worst(got, want, bound)[1] <= 1.0


def _ulp_noise(want, seed):
    """want moved by one fp16 ulp at a random half of the elements: what a kernel that rounds its (fp32) result to
    the other neighbour of the same exact value stores."""
    g = torch.Generator().manual_seed(seed)
    sign = torch.randint(0, 3, want.shape, generator=g).double() - 1
    return R.f16(want + sign * R.ulp16(want))


def _h(shape, scale, g):
    return (torch.randn(*shape, generator=g) * scale).half().double()


def _stream_weights(cin, mid, g):
    w1 = _h((mid, cin), (2.0 / cin) ** 0.5, g)
    b1 = torch.randn(mid, generator=g) * 0.05
    pws = [(_h((mid, mid), (1.0 / mid) ** 0.5, g), torch.randn(mid, generator=g) * 0.05) for _ in range(10)]
    dws = [(_h((9, mid), (2.0 / 9) ** 0.5, g), torch.randn(mid, generator=g) * 0.05) for _ in range(10)]
    return w1, b1, pws, dws


def test_streams_bound_admits_rounding_and_rejects_halo_crop_and_group_faults():
    """Kernel S at the stage-1 cluster geometry (four 16-row strips): a tail off by one ulp passes; a strip's first
    row computed from a stale halo row, the last crop replaced by its neighbour, or one 8-channel group taken from
    another group fails."""
    g = torch.Generator().manual_seed(3)
    n, h, w, cin, mid = 6, 64, 32, 64, 64
    x = (torch.randn(n, h, w, cin, generator=g).abs() * 0.7).half().double()
    w1, b1, pws, dws = _stream_weights(cin, mid, g)
    tails = R.osb_streams(x, w1, b1, pws, dws)
    want, bound = tails[3]
    assert _passes(_ulp_noise(want, 1), want, bound)
    bad = want.clone()                       # the depthwise of strip 1's first row read the previous level's halo
    bad[2, 16] = want[2, 15]
    assert not _passes(bad, want, bound)
    bad = want.clone()
    bad[n - 1] = want[n - 2]
    assert not _passes(bad, want, bound)
    bad = want.clone()
    bad[..., 8:16] = want[..., 0:8]
    assert not _passes(bad, want, bound)
    # strip sums: a strip missing from the sums is far outside the fp32 summation bound
    sums, sb = R.strip_sums([t for t, _ in tails], 4)
    assert _passes(sums.float().double(), sums, sb)
    bad = sums.clone()
    bad[:, 0] = 0
    assert not _passes(bad, sums, sb)


def _merge_case(g, n=4, h=16, w=8, mid=128, cout=512, cin=384):
    tails = [(torch.randn(n, h, w, mid, generator=g).abs() * 0.6).half().double() for _ in range(4)]
    gap = torch.stack([torch.stack([t[:, :h // 2].sum((1, 2)), t[:, h // 2:].sum((1, 2))], 1) for t in tails], 2)
    gap = gap.float().double()                                        # (n, strips, 4, mid) fp32
    cr = mid // 16
    gw = (torch.randn(cr, mid, generator=g) * (2.0 / mid) ** 0.5, torch.randn(cr, generator=g) * 0.1,
          torch.randn(mid, cr, generator=g) * (2.0 / cr) ** 0.5, torch.randn(mid, generator=g) * 0.1)
    gw = tuple(a.float().double() for a in gw)
    w3 = _h((cout, mid), (1.0 / mid) ** 0.5, g)
    wd = _h((cout, cin), (1.0 / cin) ** 0.5, g)
    bias = (torch.randn(cout, generator=g) * 0.05).float().double()
    x = (torch.randn(n, h, w, cin, generator=g).abs() * 0.7).half().double()
    return tails, gap, gw, w3, wd, bias, x


def test_streams_reference_is_the_composition_of_its_ops():
    """Kernel S's reference equals conv1 followed, per stream, by its chain of pointwise + depthwise ops, each from
    x1 and each rounded to fp16 (the single-op functions)."""
    g = torch.Generator().manual_seed(4)
    x = (torch.randn(2, 16, 8, 128, generator=g).abs()).half().double()
    w1, b1, pws, dws = _stream_weights(128, 128, g)
    tails = R.osb_streams(x, w1, b1, pws, dws)
    x1 = R.conv(x, w1[:, None, None, :], b1, act='relu')[0]
    lvl = 0
    for s in range(4):
        cur = x1
        for _ in range(s + 1):
            cur = R.conv(cur, pws[lvl][0][:, None, None, :], pws[lvl][1])[0]
            cur = R.dw(cur, dws[lvl][0], dws[lvl][1], 'relu', 'chain9')[0]
            lvl += 1
        assert torch.equal(tails[s][0], cur), s


def test_merge_bound_admits_rounding_and_rejects_gate_and_k_slice_faults():
    """Kernel G with a downsample: one ulp passes; one gate value of one crop taken from another channel, a strip
    missing from the gate's sums, or one 64-wide K slice of the downsample left out fails."""
    g = torch.Generator().manual_seed(5)
    tails, gap, gw, w3, wd, bias, x = _merge_case(g)
    want, bound = R.osb_merge(tails, gap, gw, w3, bias, x=x, wd=wd)
    assert _passes(_ulp_noise(want, 2), want, bound)
    # one gate value: crop 3, stream 1, channel 5 reads channel 6's gate
    m, em = R.strip_mean(gap, 16 * 8)
    gv, eg = R.gate_vector(m, em, *gw)
    gv2 = gv.clone()
    gv2[1, 3, 5] = gv[1, 3, 6]
    u, _ = R.gate4_apply(tails, gv2, eg)
    bad = R.f16((u @ w3.t() + x @ wd.t() + bias).clamp_min(0))
    assert not _passes(bad, want, bound)
    # the gate summed from strip 1 only
    bad, _ = R.osb_merge(tails, torch.cat([torch.zeros_like(gap[:, :1]), gap[:, 1:]], 1), gw, w3, bias, x=x, wd=wd)
    assert not _passes(bad, want, bound)
    # K slice 64..127 of the downsample dropped
    wd2 = wd.clone()
    wd2[:, 64:128] = 0
    bad, _ = R.osb_merge(tails, gap, gw, w3, bias, x=x, wd=wd2)
    assert not _passes(bad, want, bound)


def test_conv_and_gate_bounds_admit_rounding_and_reject_faults():
    g = torch.Generator().manual_seed(9)
    n, h, w, cin, cout = 40, 8, 8, 128, 64
    x = (torch.randn(n, h, w, cin, generator=g) * 0.5).half().double()
    wt = _h((cout, 1, 1, cin), (2.0 / cin) ** 0.5, g)
    b = (torch.randn(cout, generator=g) * 0.1).float().double()
    res = (torch.randn(n, h, w, cout, generator=g).abs()).half().double()
    want, bound = R.conv(x, wt, b, act='relu', res=res, res_first=True)
    assert _passes(_ulp_noise(want, 3), want, bound)
    wt2 = wt.clone()
    wt2[..., 64:] = 0                                                  # second K slice of 64 dropped
    assert not _passes(R.conv(x, wt2, b, act='relu', res=res)[0], want, bound)
    assert not _passes(R.conv(x, wt, b, act='relu', res=res, res_first=False)[0], want, bound)   # Darknet order
    bad = want.clone()
    bad[n - 1] = want[n - 3]                                           # a crop at a high batch index
    assert not _passes(bad, want, bound)
    bad = want.clone()
    bad[..., 16:24] = want[..., 8:16]                                  # one 8-channel group
    assert not _passes(bad, want, bound)
    # channel gate: one gate value
    c = 16
    xs = (torch.randn(n, h, w, c, generator=g).abs()).half().double()
    gw = tuple(a.float().double() for a in (torch.randn(4, c, generator=g) * 0.5, torch.randn(4, generator=g) * 0.1,
                                            torch.randn(c, 4, generator=g) * 0.7, torch.randn(c, generator=g) * 0.1))
    want, bound = R.gate(xs, gw)
    assert _passes(_ulp_noise(want, 4), want, bound)
    m, em = R.channel_mean(xs)
    gv, _ = R.gate_vector(m, em, *gw)
    gv[n - 1, 3] = gv[n - 1, 4]
    assert not _passes(R.f16(xs * gv[:, None, None, :]), want, bound)


def test_avgpool_and_maxpool_bounds():
    g = torch.Generator().manual_seed(2)
    x = torch.randn(3, 8, 4, 16, generator=g).half().double()
    want, bound = R.avgpool2(x)
    assert _passes(_ulp_noise(want, 5), want, bound)
    assert not _passes(R.f16(want / 0.25 * 0.24), want, bound)
    want, bound = R.maxpool3s2(x)
    assert float(bound.abs().max()) == 0.0
    assert want.shape == (3, 4, 2, 16)
