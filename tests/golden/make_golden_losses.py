"""Generate tests/golden/losses.npz by executing the REFERENCE'S OWN loss code (`embodiedscan/models/losses/
chamfer_distance.py` and `FCAF3DHeadRotMat.loss_by_feat`, imported in place through make_golden's stubs) on the seeded
inputs of loss_cases.py. It writes only that one fixture:

    python tests/golden/make_golden_losses.py

Stored per case: the inputs, the loss values, the arg-minimum indices and the autograd gradients. For 'none' reductions
the gradient is that of sum(loss * cotangent) with a stored seeded cotangent.
"""
import os
import sys

import torch

HERE = os.path.dirname(os.path.abspath(__file__))
if HERE not in sys.path:
    sys.path.insert(0, HERE)

import make_golden  # noqa: E402  (installs the reference stubs)
from cases import target_cases  # noqa: E402
from loss_cases import (GROUPS, HEAD_GRID, MODES, REDUCTIONS, bbox_cases, chamfer_cases, head_config_name,  # noqa: E402
                        head_loss_inputs)


def _cotangent(shape, seed):
    return torch.rand(shape, generator=torch.Generator().manual_seed(seed)) + 0.5


def _backward(loss, seed):
    """Scalar: loss.backward(); tensor: sum(loss * cotangent). Returns the cotangent used (or None)."""
    if loss.dim() == 0:
        loss.backward()
        return None
    cot = _cotangent(loss.shape, seed)
    (loss * cot).sum().backward()
    return cot


def gen_chamfer(out):
    from embodiedscan.models.losses.chamfer_distance import ChamferDistance, chamfer_distance
    for name, c in chamfer_cases().items():
        out[f'cd/{name}/src'], out[f'cd/{name}/dst'] = c['src'], c['dst']
        for k in ('src_weight', 'dst_weight'):
            out[f'cd/{name}/{k}'] = c[k] if torch.is_tensor(c[k]) else torch.tensor(float(c[k]))
        for mode in MODES:
            for red in REDUCTIONS:
                key = f'cd/{name}/{mode}/{red}'
                src = c['src'].clone().requires_grad_(True)
                dst = c['dst'].clone().requires_grad_(True)
                ls, ld, i1, i2 = chamfer_distance(src, dst, c['src_weight'], c['dst_weight'], mode, red)
                out[f'{key}/loss_src'], out[f'{key}/loss_dst'] = ls, ld
                out[f'{key}/idx1'], out[f'{key}/idx2'] = i1, i2
                if red == 'none':
                    cs, cd_ = _cotangent(ls.shape, 1), _cotangent(ld.shape, 2)
                    ((ls * cs).sum() + (ld * cd_).sum()).backward()
                    out[f'{key}/cot_src'], out[f'{key}/cot_dst'] = cs, cd_
                else:
                    (ls + 0.5 * ld).backward()
                out[f'{key}/grad_src'], out[f'{key}/grad_dst'] = src.grad, dst.grad
                # the registered module: loss_src_weight / loss_dst_weight, reduction_override, return_indices
                mod = ChamferDistance(mode=mode, reduction='mean', loss_src_weight=0.6, loss_dst_weight=1.5)
                m = mod(c['src'], c['dst'], c['src_weight'], c['dst_weight'], reduction_override=red, return_indices=True)
                out[f'{key}/module_src'], out[f'{key}/module_dst'] = m[0], m[1]


def gen_bbox(out):
    from embodiedscan.models.losses.chamfer_distance import BBoxCDLoss, bbox_to_corners
    for dim, (src0, tgt, w) in bbox_cases(bbox_to_corners).items():
        out[f'bbox/{dim}/source'], out[f'bbox/{dim}/target'] = src0, tgt
        out[f'bbox/{dim}/weight'] = w if torch.is_tensor(w) else torch.tensor(float(w))
        for mode in MODES:
            for group in GROUPS:
                for red in REDUCTIONS:
                    key = f'bbox/{dim}/{mode}/{group}/{red}'
                    src = src0.clone().requires_grad_(True)
                    loss = BBoxCDLoss(mode=mode, group=group, reduction=red, loss_weight=1.3)(src, tgt, loss_weight=w)
                    out[f'{key}/loss'] = loss
                    cot = _backward(loss, 3)
                    if cot is not None:
                        out[f'{key}/cot'] = cot
                    out[f'{key}/grad'] = src.grad


def gen_head(out):
    from embodiedscan.models.dense_heads.fcaf3d_head import FCAF3DHeadRotMat
    from embodiedscan.structures import EulerDepthInstance3DBoxes
    from mmengine.structures import InstanceData
    points, center, bbox, cls, gts = head_loss_inputs(target_cases)
    # the inputs are not stored: tests regenerate them with loss_cases.head_loss_inputs (checked by a checksum)
    out['head/in/checksum'] = torch.tensor([sum(float(t.double().sum()) for lv in x for t in lv)
                                            for x in (points, center, bbox, cls)], dtype=torch.float64)
    weights = {0: None, 3: [0.25, 0.35, 0.4], 4: [0.2, 0.2, 0.2, 0.4]}
    for mode, group, norm, dec in HEAD_GRID:
        head = FCAF3DHeadRotMat(num_classes=284, in_channels=(8, 16, 32, 64), out_channels=8, num_reg_outs=12,
                                voxel_size=.01, pts_prune_threshold=1000, pts_assign_threshold=27,
                                pts_center_threshold=18, bbox_loss=dict(type='BBoxCDLoss', mode=mode, group=group,
                                                                        loss_weight=1.0),
                                decouple_bbox_loss=dec > 0, decouple_groups=dec if dec else 3,
                                decouple_weights=weights[dec], norm_decouple_loss=norm)
        bb = [[t.clone().requires_grad_(True) for t in lv] for lv in bbox]
        insts = []
        for boxes, labels in gts:
            inst = InstanceData()
            inst.bboxes_3d = EulerDepthInstance3DBoxes(boxes.clone(), box_dim=9, origin=(.5, .5, .5))
            inst.labels_3d = labels.clone()
            insts.append(inst)
        losses = head.loss_by_feat(center, bb, cls, points, insts, [{}, {}])
        losses['loss_bbox'].backward()
        key = f'head/{head_config_name(mode, group, norm, dec)}'
        for k in ('loss_center', 'loss_bbox', 'loss_cls'):
            out[f'{key}/{k}'] = losses[k]
        out[f'{key}/grad_bbox'] = torch.cat([bb[l][b].grad for l in range(4) for b in range(2)])
    # reference targets per scan (levels concatenated), for CPU runs of the ATen fallback
    for b, (boxes, labels) in enumerate(gts):
        c, t, k = head.get_targets([points[l][b] for l in range(4)],
                                   EulerDepthInstance3DBoxes(boxes.clone(), box_dim=9, origin=(.5, .5, .5)), labels)
        out[f'head/targets/{b}/center'], out[f'head/targets/{b}/bbox'], out[f'head/targets/{b}/cls'] = c, t, k
        print('head scan', b, 'positives', int((k >= 0).sum()))


if __name__ == '__main__':
    torch.manual_seed(0)
    torch.set_num_threads(8)
    out = {}
    gen_chamfer(out)
    gen_bbox(out)
    gen_head(out)
    make_golden.save('losses', **out)
