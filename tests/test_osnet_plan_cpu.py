"""CPU: the launch plan of the OSNet engine (engine.plan_osnet) and the op shapes it is computed from.  Every op list
the engine runs is cut into launch groups that cover each op exactly once, in order, with the fused kernels taken
exactly where their shapes allow."""
import pytest

from fastmot_b200.engine import plan_osnet
from fastmot_b200.models import onnx_io, osnet
from fastmot_b200.models.onnx_import import export_reid_onnx, import_reid_onnx


def _plan(lib, ops, hw=(256, 128), fuse_osb=True):
    plan = plan_osnet(ops, hw, fuse_osb, lib)
    assert [k for g in plan for k in g.ops] == list(range(len(ops)))
    return plan


def _kinds(plan):
    return [g.kind for g in plan]


def test_x1_fused_plan(lib):
    ops = osnet.build_osnet(1.0)
    plan = _plan(lib, ops)
    stage = ['S', 'G', 'S', 'G']
    assert _kinds(plan) == ['stem'] + stage + ['conv', 'avgpool2'] + stage + ['conv', 'avgpool2'] + stage + \
        ['conv', 'gap', 'fc']
    s = [g for g in plan if g.kind == 'S']
    g_ = [g for g in plan if g.kind == 'G']
    assert [g.info['strips'] for g in s] == [4, 4, 2, 2, 1, 1]
    assert [g.info['ncta'] for g in g_] == [128, 128, 96, 96, 128, 128]
    # each S group ends right before the gate4 over its tails, which G starts with; G ends with the residual add
    for a, b in zip(s, g_):
        assert b.ops[0] == a.ops[-1] + 1 and tuple(ops[b.ops[0]][3]) == tuple(a.info['tails'])
        assert ops[b.ops[-1]][0] == 'add_relu' and b.info['add'] is ops[b.ops[-1]]
    assert [g.info['ds'] is not None for g in g_] == [True, False] * 3


def test_x1_per_layer_plan(lib):
    plan = _plan(lib, osnet.build_osnet(1.0), fuse_osb=False)
    kinds = _kinds(plan)
    assert kinds.count('conv+add') == 6 and kinds.count('gate4') == 6 and kinds.count('maxpool3s2') == 1
    assert not {'stem', 'S', 'G', 'gate4_pooled'} & set(kinds)


def test_x025_plan(lib):
    kinds = _kinds(_plan(lib, osnet.build_osnet(0.25)))
    assert kinds.count('conv+add') == 6 and kinds.count('gate4') == 6
    assert not {'stem', 'S', 'G', 'gate4_pooled'} & set(kinds)


@pytest.mark.parametrize("ch", [64, 10])
def test_custom_graph_plan(lib, ch):
    from test_onnx_import import _custom_graph
    ops, _, in_shape, _ = import_reid_onnx(onnx_io.serialize(_custom_graph(ch)))
    kinds = _kinds(_plan(lib, ops, in_shape[1:]))
    assert kinds == ['conv', 'maxpool3s2', 'conv', 'dw', 'add_relu', 'conv', 'conv', 'gate', 'gate', 'conv', 'avgpool2',
                     'gap', 'fc'], kinds


def test_imported_osnet_plans_like_the_built_in_one(lib):
    ops = osnet.build_osnet(1.0)
    w = osnet.synthetic_weights(ops, calibrate=False)
    ops2, _, in_shape, _ = import_reid_onnx(onnx_io.serialize(export_reid_onnx(ops, w)))
    assert _kinds(_plan(lib, ops2, in_shape[1:])) == _kinds(_plan(lib, ops))


def test_shapes_and_macs():
    ops = osnet.build_osnet(1.0)
    shapes = osnet.infer_shapes(ops, 256, 128)
    assert len(shapes) == len(ops)
    assert shapes[:2] == [(64, 128, 64), (64, 64, 32)]          # the stem binds 'x' twice: per op, not per name
    assert shapes[-3:] == [(512, 16, 8), (512, 1, 1), (512, 1, 1)]
    assert osnet.count_macs(ops) == 978_845_696
    assert osnet.count_macs(osnet.build_osnet(0.25)) == 82_313_216
