"""CPU: the float64 rotated 3D IoU oracle (oracle/rotiou_ref.py) against closed forms, finite differences and the
reference's RotatedIoU3DLoss / FCAF3DHead (tests/golden/fcaf3d_iou.npz); building FCAF3DHead and RotatedIoU3DLoss from
config dicts, through MODELS and through the reference's registry, with the reference's parameter names and shapes."""
import math
import os
import sys
import types

import numpy as np
import pytest
import torch

from rotiou_util import R, random_pairs

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden')
if GOLD not in sys.path:
    sys.path.insert(0, GOLD)

from fcaf3d_cases import AVG_FACTORS, HEAD_CASES, HEAD_CFG, REDUCTIONS, WEIGHTS, iou_weight  # noqa: E402


def golden():
    return np.load(os.path.join(GOLD, 'fcaf3d_iou.npz'))


def box(x=0., y=0., z=0., w=1., l=1., h=1., a=0.):
    return torch.tensor([[x, y, z, w, l, h, a]], dtype=torch.float64)


def iou(a, b):
    return float(R.diff_iou_rotated_3d(a, b)[0])


def test_identical_boxes():
    b = box(0.3, -1.2, 0.8, 1.4, 0.6, 0.9, 0.7)
    assert iou(b, b) == pytest.approx(1.0, abs=1e-12)


def test_axis_aligned_pairs_are_products_of_interval_overlaps():
    a, b = box(0, 0, 0, 2, 1, 1, 0), box(0.5, 0.25, 0.2, 1, 2, 1, 0)
    ox, oy, oz = 1.0, 1.0, 0.8                           # [-1,1]x[-.5,.5]x[-.5,.5] vs [0,1]x[-.75,1.25]x[-.3,.7]
    inter = ox * oy * oz
    assert iou(a, b) == pytest.approx(inter / (2 + 2 - inter), rel=1e-12)


def test_square_against_itself_turned_45_degrees():
    s = 2 * (math.sqrt(2) - 1)                           # the regular octagon of the two unit squares
    assert iou(box(), box(a=math.pi / 4)) == pytest.approx(s / (2 - s), rel=1e-12)
    assert s / (2 - s) == pytest.approx(1 / math.sqrt(2), rel=1e-12)


@pytest.mark.parametrize('other', [box(x=3.0), box(y=-1.5, a=0.3), box(z=1.5), box(z=-2.0, a=1.0)])
def test_disjoint_in_bev_or_z(other):
    assert iou(box(), other) == 0.0


def test_containment_is_the_volume_ratio():
    outer, inner = box(0, 0, 0, 3, 2, 2, 0.4), box(0.2, -0.1, 0.1, 1, 0.5, 1, 1.3)
    assert iou(outer, inner) == pytest.approx((1 * 0.5 * 1) / (3 * 2 * 2), rel=1e-12)
    assert iou(inner, outer) == pytest.approx((1 * 0.5 * 1) / (3 * 2 * 2), rel=1e-12)


def test_oracle_gradients_match_central_differences():
    a, b = random_pairs(64, 3)
    a, b = a.double(), b.double()
    _, ga, gb = R.iou_and_grads(a, b)
    h = 1e-6
    for x, g in ((a, ga), (b, gb)):
        num = torch.zeros_like(g)
        for c in range(7):
            xp, xm = x.clone(), x.clone()
            xp[:, c] += h
            xm[:, c] -= h
            args_p = (xp, b) if x is a else (a, xp)
            args_m = (xm, b) if x is a else (a, xm)
            num[:, c] = (R.diff_iou_rotated_3d(*args_p) - R.diff_iou_rotated_3d(*args_m)) / (2 * h)
        assert float((num - g).abs().max()) <= 1e-6


def test_population_stays_out_of_the_degeneracy_band():
    a, b = random_pairs(2000, 0)
    assert float(R.degeneracy_margin(a, b).min()) >= 1e-4
    v = R.diff_iou_rotated_3d(a.double(), b.double())
    assert 0.5 < float((v > 0).double().mean()) < 0.95, 'the population must mix overlapping and disjoint pairs'


@pytest.mark.parametrize('wk,red,af', [(wk, red, af) for wk in WEIGHTS for red in REDUCTIONS for af in AVG_FACTORS
                                        if af is None or red != 'sum'])      # avg_factor with 'sum' is an error
def test_oracle_loss_matches_reference(wk, red, af):
    """weight_reduce_loss on the float64 oracle IoU against the reference's RotatedIoU3DLoss, every reduction x weight x
    avg_factor: the same reduction rules the CUDA module applies (tests/test_rotiou_gpu.py)."""
    from embodiedscan_b200.dense_heads import weight_reduce_loss
    z = golden()
    key = f'loss/{wk}/{red}/{"af" if af else "none"}'
    pred = torch.from_numpy(z['loss/pred'])
    target = torch.from_numpy(z['loss/target'])
    w = iou_weight(wk, len(target))
    if w is not None and not torch.any(w > 0):
        got = pred.sum() * w.sum()
    else:
        if w is not None and w.dim() > 1:
            w = w.mean(-1)
        got = 1.7 * weight_reduce_loss(1 - R.diff_iou_rotated_3d(pred.double(), target.double()).float(), w, red, af)
    want = torch.from_numpy(z[f'{key}/loss'])
    assert got.shape == want.shape
    assert torch.allclose(got.double(), want.double(), rtol=1e-6, atol=1e-7)


def test_rotation_in_axis_2_matches_reference_convention():
    """The decode of a 7-channel prediction rotates the centre shift counter-clockwise (x' = x cos - y sin): the
    reference's decoded boxes, stored in the fixture, pin it."""
    from embodiedscan_b200 import FCAF3DHead
    from cases import target_cases
    from fcaf3d_cases import head_inputs
    z = golden()
    for name, (n_reg, scans) in HEAD_CASES.items():
        points, _, bbox, _, _ = head_inputs(target_cases, n_reg, scans)
        for b in range(len(scans)):
            pts = torch.cat([points[l][b] for l in range(4)])
            got = FCAF3DHead._bbox_pred_to_bbox(pts, torch.cat([bbox[l][b] for l in range(4)]))
            assert torch.allclose(got, torch.from_numpy(z[f'head/{name}/decoded/{b}']), rtol=1e-6, atol=1e-6), name


def _head_cfg(n_reg, **kw):
    return dict(type='FCAF3DHead', num_reg_outs=n_reg, bbox_loss=dict(type='RotatedIoU3DLoss', loss_weight=1.0),
                **HEAD_CFG, **kw)


@pytest.mark.parametrize('n_reg', [7, 9])
def test_head_builds_from_config_with_reference_names_and_shapes(n_reg):
    from embodiedscan_b200 import MODELS, FCAF3DHead, RotatedIoU3DLoss
    head = MODELS.build(_head_cfg(n_reg))
    assert type(head) is FCAF3DHead and isinstance(head.bbox_loss, RotatedIoU3DLoss)
    z = golden()
    names = [str(n) for n in z[f'manifest/r{n_reg}/manifest_names']]
    shapes = [str(s) for s in z[f'manifest/r{n_reg}/manifest_shapes']]
    own = head.state_dict()
    assert list(own) == names
    assert [','.join(map(str, v.shape)) for v in own.values()] == shapes
    from embodiedscan_b200.checkpoint import load_reference_checkpoint
    load_reference_checkpoint(head, {'state_dict': {k: torch.zeros_like(v) for k, v in own.items()}})


def test_loss_builds_from_config():
    from embodiedscan_b200 import MODELS, RotatedIoU3DLoss
    loss = MODELS.build(dict(type='RotatedIoU3DLoss', reduction='sum', loss_weight=0.5))
    assert isinstance(loss, RotatedIoU3DLoss) and loss.reduction == 'sum' and loss.loss_weight == 0.5
    with pytest.raises(ValueError):
        RotatedIoU3DLoss(reduction='avg')


def test_default_axis_aligned_iou_loss_raises():
    """The reference's default box loss, AxisAlignedIoULoss, is registered nowhere (not in the reference either)."""
    from embodiedscan_b200 import MODELS
    cfg = _head_cfg(7)
    cfg.pop('bbox_loss')
    with pytest.raises(KeyError, match='AxisAlignedIoULoss'):
        MODELS.build(cfg)


def test_head_rejects_unsupported_options():
    from embodiedscan_b200 import MODELS
    with pytest.raises(ValueError, match='num_reg_outs'):
        MODELS.build(_head_cfg(8))
    with pytest.raises(ValueError, match='RotatedIoU3DLoss'):
        MODELS.build(dict(_head_cfg(7), bbox_loss=dict(type='BBoxCDLoss')))


def test_no_cpu_fallback():
    from embodiedscan_b200 import rotated_iou_3d
    with pytest.raises(ValueError, match='CUDA'):
        rotated_iou_3d(torch.zeros(2, 7), torch.zeros(2, 7))


def test_reference_registry_builds_esb200_fcaf3d_head(monkeypatch):
    """The drop-in path of tests/test_reference_dropin_cpu.py for a detector config that swaps in the IoU head: after
    register_into_reference() the reference's registry builds our FCAF3DHead and RotatedIoU3DLoss."""
    import refstubs
    pkg = types.ModuleType('embodiedscan')
    reg = types.ModuleType('embodiedscan.registry')
    reg.MODELS, reg.TASK_UTILS = refstubs.Registry('model'), refstubs.Registry('task util')
    pkg.registry = reg
    monkeypatch.setitem(sys.modules, 'embodiedscan', pkg)
    monkeypatch.setitem(sys.modules, 'embodiedscan.registry', reg)
    import embodiedscan_b200
    from embodiedscan_b200.registry import MODELS, TASK_UTILS, register_into_reference
    from embodiedscan_b200.synth import mv_det3d_config

    def placeholder(name):
        def init(self, *args, **kwargs):
            raise AssertionError(f'the reference class {name} was built: register_into_reference() did not override it')
        return type(name, (), {'__init__': init})

    for ours, theirs in ((MODELS, reg.MODELS), (TASK_UTILS, reg.TASK_UTILS)):
        for name in ours._module_dict:
            theirs.register_module(name=name, module=placeholder(name))
    register_into_reference()
    cfg = mv_det3d_config('C1')
    head = cfg['bbox_head']
    for k in ('decouple_bbox_loss', 'decouple_groups', 'decouple_weights'):
        head.pop(k)
    head.update(type='FCAF3DHead', num_reg_outs=9, bbox_loss=dict(type='RotatedIoU3DLoss', loss_weight=1.0))
    model = reg.MODELS.build(cfg)
    assert type(model.bbox_head) is embodiedscan_b200.FCAF3DHead
    assert type(model.bbox_head.bbox_loss) is embodiedscan_b200.RotatedIoU3DLoss
    assert reg.MODELS.build(dict(type='RotatedIoU3DLoss')).__class__ is embodiedscan_b200.RotatedIoU3DLoss
