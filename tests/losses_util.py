"""Shared helpers of the chamfer-loss tests: the golden fixture (tests/golden/losses.npz), the seeded head inputs, and a
chunked ATen restatement of the reference's chamfer_distance (chamfer_distance.py:13-79) that never holds more than a
(B, chunk, M) block of distances."""
import os
import sys

import numpy as np
import torch
import torch.nn.functional as F

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden')
if GOLD not in sys.path:
    sys.path.insert(0, GOLD)

from cases import target_cases  # noqa: E402
from loss_cases import (GROUPS, HEAD_GRID, MODES, REDUCTIONS, chamfer_cases, head_config_name,  # noqa: E402,F401
                        head_loss_inputs)

_CRIT = {'l1': F.l1_loss, 'l2': F.mse_loss, 'smooth_l1': F.smooth_l1_loss}


def golden():
    return np.load(os.path.join(GOLD, 'losses.npz'))


def tensor(z, key, device='cpu'):
    return torch.from_numpy(np.array(z[key])).to(device)


def weight(z, key, device='cpu'):
    """Stored weights: 0-d arrays are floats, anything else a tensor."""
    w = np.array(z[key])
    return float(w) if w.ndim == 0 else torch.from_numpy(w).to(device)


def nearest(q, r, mode, chunk=None, with_margin=False):
    """Per query row of q (B,N,C): min over r (B,M,C) of the criterion summed over C, its first arg-minimum and, when
    asked, the relative margin (second best - best) / max(best, 1e-6). The reference's expand, `chunk` rows at a time."""
    crit = _CRIT[mode]
    N, M = q.shape[1], r.shape[1]
    chunk = chunk or N
    dist, idx, margin = [], [], []
    for s0 in range(0, N, chunk):
        qs = q[:, s0:s0 + chunk]
        d = crit(qs[:, :, None, :].expand(-1, -1, M, -1), r[:, None].expand(-1, qs.shape[1], -1, -1),
                 reduction='none').sum(-1)
        v, i = torch.min(d, dim=2)
        dist.append(v)
        idx.append(i)
        if with_margin:
            if M > 1:
                top = torch.topk(d.detach(), 2, dim=2, largest=False).values
                margin.append((top[..., 1] - top[..., 0]) / top[..., 0].clamp(min=1e-6))
            else:
                margin.append(torch.full_like(v, float('inf')))
    out = (torch.cat(dist, 1), torch.cat(idx, 1))
    return out + (torch.cat(margin, 1), ) if with_margin else out


def chamfer_oracle(src, dst, src_weight=1.0, dst_weight=1.0, mode='l2', reduction='mean', chunk=None):
    """chamfer_distance(src, dst, src_weight, dst_weight, mode, reduction) restated with bounded memory. The criteria are
    symmetric, so the dst -> src direction is the same search with the sets swapped."""
    d1, i1 = nearest(src, dst, mode, chunk)
    d2, i2 = nearest(dst, src, mode, chunk)
    loss_src, loss_dst = d1 * src_weight, d2 * dst_weight
    if reduction == 'sum':
        loss_src, loss_dst = loss_src.sum(), loss_dst.sum()
    elif reduction == 'mean':
        loss_src, loss_dst = loss_src.mean(), loss_dst.mean()
    return loss_src, loss_dst, i1, i2


def head_inputs(device='cpu'):
    """(center, bbox, cls, points) level-major lists of per-scan tensors and the gt instances of the head cases."""
    from embodiedscan_b200.structures import EulerDepthInstance3DBoxes, InstanceData
    points, center, bbox, cls, gts = head_loss_inputs(target_cases)
    mv = lambda x: [[t.to(device) for t in lv] for lv in x]  # noqa: E731
    insts = []
    for boxes, labels in gts:
        inst = InstanceData()
        inst.bboxes_3d = EulerDepthInstance3DBoxes(boxes.clone().to(device), box_dim=9, origin=(.5, .5, .5))
        inst.labels_3d = labels.to(device)
        insts.append(inst)
    checksum = [sum(float(t.double().sum()) for lv in x for t in lv) for x in (points, center, bbox, cls)]
    return mv(center), mv(bbox), mv(cls), mv(points), insts, checksum


HEAD_WEIGHTS = {0: None, 3: [0.25, 0.35, 0.4], 4: [0.2, 0.2, 0.2, 0.4]}


def build_head(mode, group, norm, dec):
    from embodiedscan_b200 import FCAF3DHeadRotMat
    return FCAF3DHeadRotMat(num_classes=284, in_channels=(8, 16, 32, 64), out_channels=8, num_reg_outs=12,
                            voxel_size=.01, pts_prune_threshold=1000, pts_assign_threshold=27, pts_center_threshold=18,
                            bbox_loss=dict(type='BBoxCDLoss', mode=mode, group=group, loss_weight=1.0),
                            decouple_bbox_loss=dec > 0, decouple_groups=dec if dec else 3,
                            decouple_weights=HEAD_WEIGHTS[dec], norm_decouple_loss=norm)
