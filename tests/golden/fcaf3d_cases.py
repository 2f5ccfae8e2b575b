"""Seeded inputs of tests/golden/fcaf3d_iou.npz (FCAF3DHead and RotatedIoU3DLoss), shared by the generator and the
tests."""
import math

import torch

NUM_CLASSES = 284
HEAD_CFG = dict(num_classes=NUM_CLASSES, in_channels=(8, 16, 32, 64), out_channels=8, voxel_size=.01,
                pts_prune_threshold=1000, pts_assign_threshold=27, pts_center_threshold=18)
TEST_CFG = dict(nms_pre=100, iou_thr=.5, score_thr=.3)
# name -> (num_reg_outs, scans): scans are target_cases() entries; 'empty_gt' is a scan without positives
HEAD_CASES = {'r7_b1': (7, ('regular', )), 'r7_b2': (7, ('regular', 'few_points')),
              'r9_b1': (9, ('regular', )), 'r9_b2': (9, ('regular', 'empty_gt'))}
REDUCTIONS = ('none', 'mean', 'sum')
WEIGHTS = ('none', 'n', 'n1', 'zero')
AVG_FACTORS = (None, 3.7)


def iou_pairs(n=24):
    """(pred, target) (n, 7) fp32 box pairs for the loss module: overlapping jittered copies and a few disjoint ones;
    pred carries two extra columns the loss must ignore."""
    g = torch.Generator().manual_seed(404)
    t = torch.cat([torch.rand(n, 2, generator=g) * 4 - 2, torch.rand(n, 1, generator=g),
                   0.3 + torch.rand(n, 3, generator=g) * 1.5, (torch.rand(n, 1, generator=g) * 2 - 1) * math.pi], 1)
    p = t.clone()
    p[:, :3] += torch.randn(n, 3, generator=g) * 0.25 * t[:, 3:6]
    p[:, 3:6] *= torch.exp(torch.randn(n, 3, generator=g) * 0.2)
    p[:, 6] += torch.randn(n, generator=g) * 0.5
    p[-3:, 0] += 10.0
    return torch.cat([p, torch.randn(n, 2, generator=g)], 1), t


def iou_weight(kind, n):
    g = torch.Generator().manual_seed(405)
    if kind == 'none':
        return None
    if kind == 'zero':
        return torch.zeros(n, 1)
    w = torch.rand(n, generator=g) + 0.1
    return w if kind == 'n' else w[:, None]


def head_inputs(target_cases, num_reg_outs, scans):
    """Level-major lists of per-scan points / centre / box-regression (6 face distances + yaw or Euler angles) / class
    predictions and the (boxes (n, 9), labels) of each scan."""
    g = torch.Generator().manual_seed(707 + num_reg_outs)
    tc = target_cases()
    points = [[tc[s][0][l].clone() for s in scans] for l in range(4)]
    center, bbox, cls = [], [], []
    for l in range(4):
        center.append([torch.randn(len(p), 1, generator=g) for p in points[l]])
        bbox.append([torch.cat([0.2 + torch.rand(len(p), 6, generator=g),
                                0.5 * torch.randn(len(p), num_reg_outs - 6, generator=g)], 1) for p in points[l]])
        cls.append([torch.randn(len(p), NUM_CLASSES, generator=g) - 2 for p in points[l]])
    gts = [(tc[s][1], tc[s][2]) for s in scans]
    return points, center, bbox, cls, gts


def checksum(points, center, bbox, cls):
    return torch.tensor([sum(float(t.double().sum()) for lv in x for t in lv) for x in (points, center, bbox, cls)],
                        dtype=torch.float64)
