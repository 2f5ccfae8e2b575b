"""CPU: the chamfer-loss family against tests/golden/losses.npz, values made by the reference's own
chamfer_distance.py and FCAF3DHeadRotMat.loss_by_feat (tests/golden/make_golden_losses.py).

  * the chunked ATen restatement of chamfer_distance (tests/losses_util.py), every case x mode x reduction;
  * BBoxCDLoss (ATen), every box width x mode x group x reduction, with float and tensor weights;
  * the ATen fallback of FCAF3DHeadRotMat's box loss, every mode x group x norm_decouple_loss x decoupling;
  * GroundingHead's batched box loss against the reference's per-layer formulation on BBoxCDLoss;
  * the option checks.
Values agree to fp32 round-off (1e-5 relative), indices exactly, gradients to 1e-5 of the tensor's largest entry."""
import pytest
import torch

from losses_util import (GROUPS, HEAD_GRID, MODES, REDUCTIONS, build_head, chamfer_oracle, golden, head_config_name,
                         head_inputs, tensor, weight)

CD_CASES = ('c3_float', 'c2_tensor', 'n1', 'duplicates')


def _close(got, want, rel=1e-5):
    got, want = got.detach().double(), want.double()
    assert got.shape == want.shape
    scale = want.abs().clamp(min=1e-6)
    assert ((got - want).abs() <= rel * scale + 1e-7).all(), float(((got - want).abs() / scale).max())


def _grad_close(got, want, tol=1e-5):
    got, want = got.detach().double(), want.double()
    assert got.shape == want.shape
    assert float((got - want).abs().max()) <= tol * max(float(want.abs().max()), 1e-12)


@pytest.mark.parametrize('case', CD_CASES)
@pytest.mark.parametrize('mode', MODES)
@pytest.mark.parametrize('reduction', REDUCTIONS)
def test_chamfer_oracle_matches_reference(case, mode, reduction):
    z = golden()
    key = f'cd/{case}/{mode}/{reduction}'
    src = tensor(z, f'cd/{case}/src').requires_grad_(True)
    dst = tensor(z, f'cd/{case}/dst').requires_grad_(True)
    ls, ld, i1, i2 = chamfer_oracle(src, dst, weight(z, f'cd/{case}/src_weight'), weight(z, f'cd/{case}/dst_weight'),
                                    mode, reduction, chunk=7)
    _close(ls, tensor(z, f'{key}/loss_src'))
    _close(ld, tensor(z, f'{key}/loss_dst'))
    assert torch.equal(i1, tensor(z, f'{key}/idx1')) and torch.equal(i2, tensor(z, f'{key}/idx2'))
    if reduction == 'none':
        ((ls * tensor(z, f'{key}/cot_src')).sum() + (ld * tensor(z, f'{key}/cot_dst')).sum()).backward()
    else:
        (ls + 0.5 * ld).backward()
    _grad_close(src.grad, tensor(z, f'{key}/grad_src'))
    _grad_close(dst.grad, tensor(z, f'{key}/grad_dst'))


@pytest.mark.parametrize('dim', (6, 7, 9))
@pytest.mark.parametrize('mode', MODES)
@pytest.mark.parametrize('group', GROUPS)
@pytest.mark.parametrize('reduction', REDUCTIONS)
def test_bbox_cd_loss_matches_reference(dim, mode, group, reduction):
    from embodiedscan_b200 import BBoxCDLoss
    z = golden()
    key = f'bbox/{dim}/{mode}/{group}/{reduction}'
    src = tensor(z, f'bbox/{dim}/source').requires_grad_(True)
    loss_fn = BBoxCDLoss(mode=mode, group=group, reduction='mean', loss_weight=1.3)
    loss = loss_fn(src, tensor(z, f'bbox/{dim}/target'), loss_weight=weight(z, f'bbox/{dim}/weight'),
                   reduction_override=reduction)
    _close(loss, tensor(z, f'{key}/loss'))
    if reduction == 'none':
        (loss * tensor(z, f'{key}/cot')).sum().backward()
    else:
        loss.backward()
    _grad_close(src.grad, tensor(z, f'{key}/grad'))


def _reference_targets(z, points):
    """The reference's per-scan targets (levels concatenated) in the head's row order: level-major, scans within."""
    parts = {k: [] for k in ('center', 'bbox', 'cls')}
    for l in range(len(points)):
        for b in range(len(points[l])):
            off = sum(len(points[ll][b]) for ll in range(l))
            n = len(points[l][b])
            for k in parts:
                parts[k].append(tensor(z, f'head/targets/{b}/{k}')[off:off + n])
    return torch.cat(parts['center']).float(), torch.cat(parts['bbox']).float(), torch.cat(parts['cls']).long()


@pytest.mark.parametrize('mode,group,norm,dec', HEAD_GRID, ids=[head_config_name(*c) for c in HEAD_GRID])
def test_head_aten_box_loss_matches_reference(monkeypatch, mode, group, norm, dec):
    """FCAF3DHeadRotMat.loss_by_feat on CPU tensors takes the ATen fallback of the box loss. Target assignment and the
    focal loss are CUDA kernels, so the reference's targets are fed in and the classification term is left out."""
    from embodiedscan_b200 import dense_heads
    z = golden()
    center, bbox, cls, points, insts, checksum = head_inputs()
    assert checksum == pytest.approx(list(tensor(z, 'head/in/checksum')), rel=1e-12)
    targets = _reference_targets(z, points)
    monkeypatch.setattr(dense_heads, 'fcaf3d_targets_batched', lambda *a, **k: targets)
    head = build_head(mode, group, norm, dec)
    monkeypatch.setattr(head.cls_loss, 'forward', lambda pred, target, row_weight=None: pred.sum() * 0)
    bb = [[t.clone().requires_grad_(True) for t in lv] for lv in bbox]
    losses = head.loss_by_feat(center, bb, cls, points, insts)
    key = f'head/{head_config_name(mode, group, norm, dec)}'
    _close(losses['loss_bbox'], tensor(z, f'{key}/loss_bbox'))
    _close(losses['loss_center'], tensor(z, f'{key}/loss_center'))
    losses['loss_bbox'].backward()
    grad = torch.cat([bb[l][b].grad for l in range(4) for b in range(2)])
    _grad_close(grad, tensor(z, f'{key}/grad_bbox'))


def _grounding_head(mode, group, norm, dec):
    from embodiedscan_b200.grounding import GroundingHead
    return GroundingHead(num_classes=256, embed_dims=32, num_pred_layer=3, loss_bbox=dict(type='BBoxCDLoss', mode=mode,
                                                                                         group=group, loss_weight=1.7),
                         decouple_bbox_loss=dec > 0, decouple_groups=dec if dec else 3,
                         decouple_weights=[0.2, 0.2, 0.2, 0.4][:dec] if dec else None, norm_decouple_loss=norm,
                         train_cfg=None)


def _reference_grounding_box_loss(loss_bbox, pred, tgt, dec, norm, w):
    """grounding_head.py:775-818 for one decoder layer, on the (fixture-pinned) BBoxCDLoss module."""
    if not dec:
        return loss_bbox(pred, tgt)
    pc, ps, pe = pred[:, :3], pred[:, 3:6], pred[:, 6:]
    tc, ts, te = tgt[:, :3], tgt[:, 3:6], tgt[:, 6:]
    srcs = (torch.cat((pc, ts, te), -1), torch.cat((tc, ps, te), -1), torch.cat((tc, ts, pe), -1))
    if norm:
        loss = sum(w[i] * loss_bbox(s, tgt, reduction_override='none') for i, s in enumerate(srcs))
        loss = (loss / ts.norm(dim=-1)[:, None].clamp(min=0.1)).mean()
    else:
        loss = sum(w[i] * loss_bbox(s, tgt) for i, s in enumerate(srcs))
    if dec == 4:
        loss = loss + w[3] * loss_bbox(pred, tgt)
    return loss


@pytest.mark.parametrize('mode,group,norm,dec', HEAD_GRID, ids=[head_config_name(*c) for c in HEAD_GRID])
def test_grounding_box_losses_match_reference_formulation(mode, group, norm, dec):
    g = torch.Generator().manual_seed(404)
    tgt = torch.cat([torch.rand(13, 3, generator=g) * 4 - 2, 0.05 + torch.rand(13, 3, generator=g),
                     torch.randn(13, 3, generator=g) * 0.5], 1)
    tgt[0, 3:6] = 0.02                                     # a box below the 0.1 size clamp
    pred = (tgt[None] + 0.2 * torch.randn(3, 13, 9, generator=g)).requires_grad_(True)
    head = _grounding_head(mode, group, norm, dec)
    got = head._box_losses(pred, tgt)
    pred_ref = pred.detach().clone().requires_grad_(True)
    want = [_reference_grounding_box_loss(head.loss_bbox, pred_ref[l], tgt, dec, norm, head.decouple_weights)
            for l in range(3)]
    for a, b in zip(got, want):
        _close(a, b.detach())
    sum(got).backward()
    sum(want).backward()
    _grad_close(pred.grad, pred_ref.grad)


def test_option_errors():
    from embodiedscan_b200 import BBoxCDLoss, ChamferDistance, chamfer_distance
    with pytest.raises(ValueError, match='mode'):
        BBoxCDLoss(mode='l3')
    with pytest.raises(ValueError, match='group'):
        BBoxCDLoss(group='g2')
    with pytest.raises(ValueError, match='reduction'):
        ChamferDistance(reduction='max')
    with pytest.raises(ValueError, match="reduction='mean'"):
        build_head_with_reduction('sum')
    with pytest.raises(ValueError, match="reduction='mean'"):
        _grounding_head_with_reduction('none')
    pts = torch.rand(1, 4, 3)
    with pytest.raises(ValueError, match='CUDA'):
        chamfer_distance(pts, pts)
    with pytest.raises(NotImplementedError):
        chamfer_distance(pts, pts, criterion_mode='l4')


def build_head_with_reduction(reduction):
    from embodiedscan_b200 import FCAF3DHeadRotMat
    return FCAF3DHeadRotMat(num_classes=4, in_channels=(8, 16), out_channels=8, num_reg_outs=12, voxel_size=.01,
                            pts_prune_threshold=1000, pts_assign_threshold=27, pts_center_threshold=18,
                            bbox_loss=dict(type='BBoxCDLoss', mode='l1', group='g8', reduction=reduction))


def _grounding_head_with_reduction(reduction):
    from embodiedscan_b200.grounding import GroundingHead
    return GroundingHead(num_classes=256, embed_dims=32, num_pred_layer=2, train_cfg=None,
                         loss_bbox=dict(type='BBoxCDLoss', mode='l2', reduction=reduction))


def test_default_bbox_cd_loss_builds_from_a_bare_config():
    """dict(type='BBoxCDLoss') builds the reference's default: mode 'l2', group 'g8', reduction 'mean'."""
    from embodiedscan_b200.registry import MODELS
    loss = MODELS.build(dict(type='BBoxCDLoss'))
    assert (loss.mode, loss.group, loss.reduction, loss.loss_weight) == ('l2', 'g8', 'mean', 1.0)
    assert MODELS.build(dict(type='ChamferDistance')).mode == 'l2'
