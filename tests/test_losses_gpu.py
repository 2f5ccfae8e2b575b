"""GPU: the chamfer-loss family on its kernels (csrc/chamfer.cu, csrc/head.cu::bbox_cd_loss_kernel) against
tests/golden/losses.npz (the reference's own values) and against the chunked ATen restatement at scale."""
import pytest
import torch

from losses_util import (GROUPS, HEAD_GRID, MODES, REDUCTIONS, build_head, golden, head_config_name, head_inputs,
                         nearest, tensor, weight)

pytestmark = pytest.mark.gpu
CD_CASES = ('c3_float', 'c2_tensor', 'n1', 'duplicates')


def _rel_close(got, want, rel):
    got, want = got.detach().double().cpu(), want.double().cpu()
    assert got.shape == want.shape
    assert ((got - want).abs() <= rel * want.abs().clamp(min=1e-6) + 1e-7).all(), \
        float(((got - want).abs() / want.abs().clamp(min=1e-6)).max())


def _grad_close(got, want, tol=1e-4):
    got, want = got.detach().double().cpu(), want.double().cpu()
    assert got.shape == want.shape
    assert float((got - want).abs().max()) <= tol * max(float(want.abs().max()), 1e-12)


@pytest.mark.parametrize('case', CD_CASES)
@pytest.mark.parametrize('mode', MODES)
@pytest.mark.parametrize('reduction', REDUCTIONS)
def test_chamfer_distance_matches_reference(case, mode, reduction):
    from embodiedscan_b200 import ChamferDistance, chamfer_distance
    z = golden()
    key = f'cd/{case}/{mode}/{reduction}'
    src = tensor(z, f'cd/{case}/src', 'cuda').requires_grad_(True)
    dst = tensor(z, f'cd/{case}/dst', 'cuda').requires_grad_(True)
    sw, dw = weight(z, f'cd/{case}/src_weight', 'cuda'), weight(z, f'cd/{case}/dst_weight', 'cuda')
    ls, ld, i1, i2 = chamfer_distance(src, dst, sw, dw, mode, reduction)
    _rel_close(ls, tensor(z, f'{key}/loss_src'), 1e-4)
    _rel_close(ld, tensor(z, f'{key}/loss_dst'), 1e-4)
    assert torch.equal(i1.cpu(), tensor(z, f'{key}/idx1')) and torch.equal(i2.cpu(), tensor(z, f'{key}/idx2'))
    if reduction == 'none':
        ((ls * tensor(z, f'{key}/cot_src', 'cuda')).sum() + (ld * tensor(z, f'{key}/cot_dst', 'cuda')).sum()).backward()
    else:
        (ls + 0.5 * ld).backward()
    _grad_close(src.grad, tensor(z, f'{key}/grad_src'))
    _grad_close(dst.grad, tensor(z, f'{key}/grad_dst'))
    mod = ChamferDistance(mode=mode, reduction='mean', loss_src_weight=0.6, loss_dst_weight=1.5)
    m = mod(src.detach(), dst.detach(), sw, dw, reduction_override=reduction, return_indices=True)
    assert len(m) == 4 and len(mod(src.detach(), dst.detach(), sw, dw)) == 2
    _rel_close(m[0], tensor(z, f'{key}/module_src'), 1e-4)
    _rel_close(m[1], tensor(z, f'{key}/module_dst'), 1e-4)


@pytest.mark.parametrize('mode', MODES)
def test_chamfer_distance_matches_restatement_at_scale(mode):
    """B = 4, N = M = 20000, C = 3: distances to 1e-5 relative, indices wherever the restatement's margin > 1e-6."""
    from embodiedscan_b200 import chamfer_distance
    g = torch.Generator(device='cuda').manual_seed(7)
    src = torch.rand(4, 20000, 3, device='cuda', generator=g) * 4 - 2
    dst = torch.rand(4, 20000, 3, device='cuda', generator=g) * 4 - 2
    d1, d2, i1, i2 = chamfer_distance(src, dst, criterion_mode=mode, reduction='none')
    for got_d, got_i, (q, r) in ((d1, i1, (src, dst)), (d2, i2, (dst, src))):
        want_d, want_i, margin = nearest(q, r, mode, chunk=1000, with_margin=True)
        _rel_close(got_d, want_d, 1e-5)
        sure = margin > 1e-6
        assert sure.float().mean() > 0.99
        assert torch.equal(got_i[sure], want_i[sure])


def test_chamfer_backward_is_bit_reproducible():
    from embodiedscan_b200 import chamfer_distance
    g = torch.Generator(device='cuda').manual_seed(8)
    src = (torch.rand(2, 3000, 3, device='cuda', generator=g) * 0.2).requires_grad_(True)   # dense: many shared NNs
    dst = (torch.rand(2, 5000, 3, device='cuda', generator=g) * 0.2).requires_grad_(True)
    grads = []
    for _ in range(2):
        src.grad = dst.grad = None
        ls, ld, _, _ = chamfer_distance(src, dst, criterion_mode='l2')
        (ls + ld).backward()
        grads.append((src.grad.clone(), dst.grad.clone()))
    assert torch.equal(grads[0][0], grads[1][0]) and torch.equal(grads[0][1], grads[1][1])


def test_chamfer_input_checks_and_dtypes():
    from embodiedscan_b200 import chamfer_distance
    with pytest.raises(ValueError, match='1 to 8'):
        chamfer_distance(torch.rand(1, 4, 9, device='cuda'), torch.rand(1, 5, 9, device='cuda'))
    with pytest.raises(ValueError, match='empty'):
        chamfer_distance(torch.rand(1, 0, 3, device='cuda'), torch.rand(1, 5, 3, device='cuda'))
    src = torch.rand(2, 30, 8, device='cuda', dtype=torch.bfloat16, requires_grad=True)
    dst = torch.rand(2, 20, 8, device='cuda', dtype=torch.bfloat16, requires_grad=True)
    ls, ld, _, _ = chamfer_distance(src, dst, criterion_mode='smooth_l1')
    (ls + ld).backward()
    assert src.grad.dtype == torch.bfloat16 and dst.grad.dtype == torch.bfloat16


@pytest.mark.parametrize('dim', (6, 7, 9))
@pytest.mark.parametrize('mode', MODES)
@pytest.mark.parametrize('group', GROUPS)
@pytest.mark.parametrize('reduction', REDUCTIONS)
def test_bbox_cd_loss_module_matches_reference(dim, mode, group, reduction):
    from embodiedscan_b200 import BBoxCDLoss
    z = golden()
    key = f'bbox/{dim}/{mode}/{group}/{reduction}'
    src = tensor(z, f'bbox/{dim}/source', 'cuda').requires_grad_(True)
    loss = BBoxCDLoss(mode=mode, group=group, reduction=reduction, loss_weight=1.3)(
        src, tensor(z, f'bbox/{dim}/target', 'cuda'), loss_weight=weight(z, f'bbox/{dim}/weight', 'cuda'))
    _rel_close(loss, tensor(z, f'{key}/loss'), 1e-3)
    (loss * tensor(z, f'{key}/cot', 'cuda')).sum().backward() if reduction == 'none' else loss.backward()
    _grad_close(src.grad, tensor(z, f'{key}/grad'))


def _fused_head_losses(mode, group, norm, dec):
    center, bbox, cls, points, insts, _ = head_inputs('cuda')
    head = build_head(mode, group, norm, dec).cuda()
    bb = [[t.clone().requires_grad_(True) for t in lv] for lv in bbox]
    return head.loss_by_feat(center, bb, cls, points, insts), bb


@pytest.mark.parametrize('mode,group,norm,dec', HEAD_GRID, ids=[head_config_name(*c) for c in HEAD_GRID])
def test_detector_head_fused_box_loss_matches_reference(mode, group, norm, dec):
    z = golden()
    losses, bb = _fused_head_losses(mode, group, norm, dec)
    key = f'head/{head_config_name(mode, group, norm, dec)}'
    for k in ('loss_bbox', 'loss_center', 'loss_cls'):
        _rel_close(losses[k], tensor(z, f'{key}/{k}'), 1e-3)
    losses['loss_bbox'].backward()
    _grad_close(torch.cat([bb[l][b].grad for l in range(4) for b in range(2)]), tensor(z, f'{key}/grad_bbox'))


def _launches(fn):
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    return sum(1 for e in prof.events() if e.device_type.name == 'CUDA' and 'memcpy' not in e.name.lower()
               and 'memset' not in e.name.lower())


def test_detector_head_box_loss_launch_count_is_configuration_independent():
    """Every BBoxCDLoss configuration launches as many kernels in the head's loss as the configured one (l1 / g8)."""
    counts = {}
    for mode, group, norm, dec in [('l1', 'g8', False, 4)] + [c for c in HEAD_GRID if c[3] == 4]:
        _fused_head_losses(mode, group, norm, dec)                     # warm-up
        counts[(mode, group, norm)] = _launches(lambda: _fused_head_losses(mode, group, norm, dec))
    assert len(set(counts.values())) == 1, counts


@pytest.mark.parametrize('mode,group,norm,dec', [c for c in HEAD_GRID if c[3] == 4],
                         ids=[head_config_name(*c) for c in HEAD_GRID if c[3] == 4])
def test_grounding_head_box_losses_on_gpu_match_cpu(mode, group, norm, dec):
    """The grounding head's batched box loss (ATen) computes the same on the GPU as on the CPU, where it is pinned."""
    from embodiedscan_b200.grounding import GroundingHead
    head = GroundingHead(num_classes=256, embed_dims=32, num_pred_layer=3, train_cfg=None, decouple_bbox_loss=True,
                         decouple_groups=4, decouple_weights=[0.2, 0.2, 0.2, 0.4], norm_decouple_loss=norm,
                         loss_bbox=dict(type='BBoxCDLoss', mode=mode, group=group, loss_weight=1.0))
    g = torch.Generator().manual_seed(5)
    tgt = torch.cat([torch.rand(9, 3, generator=g), 0.1 + torch.rand(9, 3, generator=g), torch.randn(9, 3, generator=g)], 1)
    pred = tgt[None] + 0.2 * torch.randn(3, 9, 9, generator=g)
    cpu = head._box_losses(pred, tgt)
    gpu = head.cuda()._box_losses(pred.cuda(), tgt.cuda())
    for a, b in zip(gpu, cpu):
        _rel_close(a, b, 1e-5)
