"""GPU: the rotated 3D IoU kernel (csrc/rotiou3d.cu) against the float64 oracle, RotatedIoU3DLoss and FCAF3DHead against
the reference (tests/golden/fcaf3d_iou.npz), bit reproducibility, and a short bf16 training run of the detector with the
IoU head.

Bounds, kernel against float64. The kernel works in fp32 relative to box A's centre on metre-sized boxes: corners carry
~1e-7 m of rounding, the shoelace sum over <= 8 vertices ~1e-6 of the area, and volumes / the union a few ulp, so the
IoU is within ~1e-6; the bound is 1e-5 absolute. A gradient is a short chain of products and quotients of those
quantities (no cancellation beyond the shoelace's), within ~1e-5 relative; the bound is 1e-4 (1 + |g|) per element.
The gradient bound holds away from degenerate configurations only: the population is drawn with a float64 margin of
1e-4 m from every vertex-inclusion, intersection and z-overlap switch (rotiou_util.random_pairs)."""
import os
import sys

import numpy as np
import pytest
import torch

from rotiou_util import R, hard_cases, iou_head_detector_config, random_pairs

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden')
if GOLD not in sys.path:
    sys.path.insert(0, GOLD)

from cases import target_cases  # noqa: E402
from fcaf3d_cases import (AVG_FACTORS, HEAD_CASES, HEAD_CFG, REDUCTIONS, TEST_CFG, WEIGHTS, checksum,  # noqa: E402
                          head_inputs, iou_weight)

pytestmark = pytest.mark.gpu
DEV = 'cuda:0'


def golden():
    return np.load(os.path.join(GOLD, 'fcaf3d_iou.npz'))


def kernel(a, b, g):
    from embodiedscan_b200 import rotated_iou_3d
    a = a.to(DEV).requires_grad_(True)
    b = b.to(DEV).requires_grad_(True)
    iou = rotated_iou_3d(a, b)
    ga, gb = torch.autograd.grad(iou, (a, b), g.to(DEV))
    return iou.detach().cpu(), ga.cpu(), gb.cpu()


def test_kernel_matches_float64_oracle_on_random_pairs():
    a, b = random_pairs(20000, 11)
    g = torch.rand(a.shape[0], generator=torch.Generator().manual_seed(2)) + 0.5
    iou, ga, gb = kernel(a, b, g)
    ri, rga, rgb = R.iou_and_grads(a, b, g)
    assert float((ri > 0).double().mean()) > 0.5
    assert float((iou.double() - ri).abs().max()) <= 1e-5
    for got, want in ((ga, rga), (gb, rgb)):
        assert torch.isfinite(got).all()
        err = (got.double() - want).abs() / (1 + want.abs())
        assert float(err.max()) <= 1e-4, float(err.max())


@pytest.mark.parametrize('name', sorted(hard_cases()))
def test_named_hard_cases(name):
    """IoU within the bound everywhere; at these degenerate configurations the gradient only has to be finite and of
    the size of the gradients around it."""
    a, b = hard_cases()[name]
    iou, ga, gb = kernel(a, b, torch.ones(a.shape[0]))
    ri, _, _ = R.iou_and_grads(a, b)
    assert float((iou.double() - ri).abs().max()) <= 1e-5, (iou, ri)
    for g in (ga, gb):
        assert torch.isfinite(g).all()
        assert float(g.abs().max()) <= 1e3 / float(torch.cat((a, b))[:, 3:6].min())


def test_row_strides_and_extra_columns():
    """7-, 9- and 12-column rows (read in place) give the same bits; columns past 7 get zero gradient."""
    from embodiedscan_b200 import rotated_iou_3d
    a, b = random_pairs(1000, 5)
    g = torch.Generator().manual_seed(6)
    ref = rotated_iou_3d(a.to(DEV), b.to(DEV))
    for extra in (2, 5):
        aw = torch.cat((a, torch.randn(a.shape[0], extra, generator=g)), 1).to(DEV).requires_grad_(True)
        bw = torch.cat((b, torch.randn(b.shape[0], extra, generator=g)), 1).to(DEV)
        got = rotated_iou_3d(aw, bw)
        assert torch.equal(got, ref)
        got.sum().backward()
        assert aw.grad.shape == aw.shape and not aw.grad[:, 7:].any()


def test_bit_identical_over_two_runs_and_finite():
    from embodiedscan_b200 import rotated_iou_3d
    a, b = random_pairs(4096, 8)
    n = 262144
    a, b = a.repeat(n // 4096, 1).to(DEV), b.repeat(n // 4096, 1).to(DEV)
    a += torch.randn(a.shape, generator=torch.Generator().manual_seed(1)).to(DEV) * 0.01
    outs = []
    for _ in range(2):
        x, y = a.clone().requires_grad_(True), b.clone().requires_grad_(True)
        iou = rotated_iou_3d(x, y)
        (iou * torch.linspace(0.5, 1.5, n, device=DEV)).sum().backward()
        outs.append((iou.detach(), x.grad, y.grad))
    for u, v in zip(*outs):
        assert torch.isfinite(u).all() and torch.equal(u, v)


@pytest.mark.parametrize('wk', WEIGHTS)
@pytest.mark.parametrize('red', REDUCTIONS)
@pytest.mark.parametrize('af', AVG_FACTORS)
def test_loss_module_matches_reference(wk, red, af):
    from embodiedscan_b200 import RotatedIoU3DLoss
    if af is not None and red == 'sum':
        with pytest.raises(ValueError):
            RotatedIoU3DLoss()(torch.zeros(2, 7, device=DEV), torch.ones(2, 7, device=DEV), avg_factor=af,
                               reduction_override=red)
        return
    z = golden()
    key = f'loss/{wk}/{red}/{"af" if af else "none"}'
    pred = torch.from_numpy(z['loss/pred']).to(DEV).requires_grad_(True)
    target = torch.from_numpy(z['loss/target']).to(DEV)
    w = iou_weight(wk, target.shape[0])
    loss = RotatedIoU3DLoss(reduction='mean', loss_weight=1.7)(pred, target, weight=None if w is None else w.to(DEV),
                                                               avg_factor=af, reduction_override=red)
    want = torch.from_numpy(z[f'{key}/loss'])
    assert loss.shape == want.shape
    assert torch.allclose(loss.detach().cpu().double(), want.double(), rtol=1e-5, atol=1e-5)
    if loss.dim() == 0:
        loss.backward()
    else:
        (loss * torch.from_numpy(z[f'{key}/cot']).to(DEV)).sum().backward()
    want_g = torch.from_numpy(z[f'{key}/grad']).double()
    assert float((pred.grad.cpu().double() - want_g).abs().max()) <= 1e-4 * (1 + float(want_g.abs().max()))


def _head_case(name):
    from embodiedscan_b200 import FCAF3DHead
    from embodiedscan_b200.structures import EulerDepthInstance3DBoxes, InstanceData
    n_reg, scans = HEAD_CASES[name]
    points, center, bbox, cls, gts = head_inputs(target_cases, n_reg, scans)
    z = golden()
    assert torch.equal(checksum(points, center, bbox, cls), torch.from_numpy(z[f'head/{name}/checksum']))
    mv = lambda x: [[t.to(DEV) for t in lv] for lv in x]  # noqa: E731
    insts = []
    for boxes, labels in gts:
        inst = InstanceData()
        inst.bboxes_3d = EulerDepthInstance3DBoxes(boxes.clone().to(DEV), box_dim=9, origin=(.5, .5, .5))
        inst.labels_3d = labels.to(DEV)
        insts.append(inst)
    head = FCAF3DHead(num_reg_outs=n_reg, bbox_loss=dict(type='RotatedIoU3DLoss'), test_cfg=TEST_CFG, **HEAD_CFG).to(DEV)
    return head, mv(points), mv(center), mv(bbox), mv(cls), insts, len(scans), z


@pytest.mark.parametrize('name', sorted(HEAD_CASES))
def test_head_losses_and_gradient_match_reference(name):
    head, points, center, bbox, cls, insts, B, z = _head_case(name)
    bb = [[t.clone().requires_grad_(True) for t in lv] for lv in bbox]
    losses = head.loss_by_feat(center, bb, cls, points, insts)
    for k in ('loss_center', 'loss_bbox', 'loss_cls'):
        got, want = float(losses[k]), float(z[f'head/{name}/{k}'])
        assert abs(got - want) <= 1e-3 * max(abs(want), 1e-6) + 1e-7, (k, got, want)
    losses['loss_bbox'].backward()
    grad = torch.cat([bb[l][b].grad for l in range(4) for b in range(B)]).cpu().double()
    want = torch.from_numpy(z[f'head/{name}/grad_bbox']).double()
    assert torch.isfinite(grad).all()
    assert float((grad - want).abs().max()) <= 1e-2 * float(want.abs().max())


@pytest.mark.parametrize('name', sorted(HEAD_CASES))
def test_head_predict_matches_reference_selection_order(name):
    head, points, center, bbox, cls, insts, B, z = _head_case(name)
    from embodiedscan_b200.structures import EulerDepthInstance3DBoxes
    with torch.no_grad():
        res = head.predict_by_feat(center, bbox, cls, points, [{'box_type_3d': EulerDepthInstance3DBoxes}] * B)
    for b, r in enumerate(res):
        labels = torch.from_numpy(z[f'head/{name}/nms/{b}/labels'])
        assert torch.equal(r.labels_3d.cpu(), labels)
        assert torch.allclose(r.scores_3d.cpu(), torch.from_numpy(z[f'head/{name}/nms/{b}/scores']), rtol=1e-3)
        boxes = torch.from_numpy(z[f'head/{name}/nms/{b}/boxes'])
        assert float((r.bboxes_3d.tensor.cpu() - boxes).abs().max()) <= 1e-3 * float(boxes.abs().max())


@pytest.mark.parametrize('n_reg', [7, 9])
def test_bf16_training_run_is_finite_and_reproducible(n_reg):
    from embodiedscan_b200 import MODELS, FCAF3DHead
    from embodiedscan_b200.engine import OptimWrapper
    from embodiedscan_b200.synth import synth_batch
    runs = []
    for _ in range(2):
        torch.manual_seed(0)
        model = MODELS.build(dict(iou_head_detector_config('C1', n_reg), compute_dtype=torch.bfloat16)).to(DEV).train()
        assert type(model.bbox_head) is FCAF3DHead
        batch = synth_batch(3, 2, n_views=2, H=240, W=320, n_points=4000)
        ow = OptimWrapper(model, lr=1e-3)
        hist = []
        for _ in range(4):
            logs = model.train_step(dict(inputs=batch['inputs'], data_samples=batch['data_samples']), ow)
            hist.append({k: float(v) for k, v in logs.items()})
        torch.cuda.synchronize()
        runs.append((hist, ow.arena.flat.detach().cpu().clone()))
    assert all(np.isfinite(v) for h in runs[0][0] for v in h.values()), runs[0][0]
    assert runs[0][0] == runs[1][0]
    assert all(h['loss_bbox'] > 0 for h in runs[0][0])
    assert torch.equal(runs[0][1], runs[1][1])
