"""Shared inputs of the rotated-IoU tests: a seeded population of box pairs kept away from degenerate configurations, and
the named hard cases."""
import math
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from oracle import rotiou_ref as R  # noqa: E402

BAND = 1e-4     # metres: pairs closer than this to a degenerate configuration are drawn again


def _draw(g, n):
    """Box A anywhere in a 6 m x 6 m room, B a jittered copy of A (overlapping most of the time), or, for one pair in
    eight, an unrelated box."""
    a = torch.empty(n, 7, dtype=torch.float64)
    a[:, :2] = torch.rand(n, 2, generator=g, dtype=torch.float64) * 6 - 3
    a[:, 2] = torch.rand(n, generator=g, dtype=torch.float64) * 2
    a[:, 3:6] = torch.exp(torch.rand(n, 3, generator=g, dtype=torch.float64) * math.log(10)) * 0.2
    a[:, 6] = (torch.rand(n, generator=g, dtype=torch.float64) * 2 - 1) * math.pi
    b = a.clone()
    b[:, :3] += torch.randn(n, 3, generator=g, dtype=torch.float64) * 0.3 * a[:, 3:6]
    b[:, 3:6] *= torch.exp(torch.randn(n, 3, generator=g, dtype=torch.float64) * 0.3)
    b[:, 6] += torch.randn(n, generator=g, dtype=torch.float64) * 0.6
    far = torch.rand(n, generator=g) < 0.125
    b[far] = _draw_free(g, int(far.sum()))
    return a, b


def _draw_free(g, n):
    b = torch.empty(n, 7, dtype=torch.float64)
    b[:, :2] = torch.rand(n, 2, generator=g, dtype=torch.float64) * 6 - 3
    b[:, 2] = torch.rand(n, generator=g, dtype=torch.float64) * 2
    b[:, 3:6] = torch.exp(torch.rand(n, 3, generator=g, dtype=torch.float64) * math.log(10)) * 0.2
    b[:, 6] = (torch.rand(n, generator=g, dtype=torch.float64) * 2 - 1) * math.pi
    return b


def random_pairs(n: int, seed: int, band: float = BAND):
    """fp32 pairs (a, b), each (n, 7), whose float64 degeneracy margin (oracle.rotiou_ref.degeneracy_margin) is at
    least `band`: a pair inside the band is drawn again (seeded, so the population is fixed)."""
    g = torch.Generator().manual_seed(seed)
    a, b = _draw(g, n)
    a, b = a.float(), b.float()
    for _ in range(50):
        bad = torch.nonzero(R.degeneracy_margin(a, b) < band).squeeze(1)
        if bad.numel() == 0:
            return a, b
        na, nb = _draw(g, bad.numel())
        a[bad], b[bad] = na.float(), nb.float()
    raise AssertionError('could not clear the degeneracy band')


def hard_cases():
    """name -> (a (k, 7), b (k, 7)) fp32: configurations at or next to the degenerate ones."""
    box = torch.tensor([0.3, -0.2, 1.0, 1.2, 0.8, 0.6, 0.4])
    c = {}
    c['identical'] = (box[None], box[None])
    shifted = box.clone()
    shifted[0] += 1.2 * math.cos(0.4)                        # shares the edge x = +w/2 of the first box
    shifted[1] += 1.2 * math.sin(0.4)
    c['shared_edge'] = (box[None], shifted[None])
    r90 = box.clone()
    r90[6] += math.pi / 2
    r180 = box.clone()
    r180[6] += math.pi
    c['rotated_90_180'] = (box[None].repeat(2, 1), torch.stack((r90, r180)))
    touch = box.clone()
    touch[0] += 1.2 * math.cos(0.4) + 1e-3 * math.cos(0.4)     # 1 mm apart
    touch[1] += 1.2 * math.sin(0.4) + 1e-3 * math.sin(0.4)
    ztouch = box.clone()
    ztouch[2] += 0.6                                          # face to face in z
    c['touching'] = (box[None].repeat(2, 1), torch.stack((touch, ztouch)))
    inner = box.clone()
    inner[3:6] *= 0.5
    inner[6] += 0.3
    c['contained'] = (box[None], inner[None])
    thin = torch.tensor([[0.0, 0.0, 0.5, 2.0, 0.01, 1.0, 0.0], [0.0, 0.0, 0.5, 2.0, 0.01, 1.0, 0.1]])
    thin_b = torch.tensor([[0.1, 0.0, 0.5, 2.0, 0.01, 1.0, 0.02], [0.0, 0.0, 0.5, 0.01, 2.0, 1.0, 0.0]])
    c['aspect_1_200'] = (thin, thin_b)
    zdis = box.clone()
    zdis[2] += 2.0
    c['z_disjoint'] = (box[None], zdis[None])
    # a square of side sqrt(2)/2 turned by 45 degrees about (1, 0): its corner (0.5, 0) lies on the unit square's edge
    on_edge = torch.tensor([1.0, 0.0, 0.0, math.sqrt(2) / 2, math.sqrt(2) / 2, 1.0, math.pi / 4])
    c['corner_on_edge'] = (torch.tensor([[0.0, 0.0, 0.0, 1.0, 1.0, 1.0, 0.0]]), on_edge[None])
    return {k: (a.float(), b.float()) for k, (a, b) in c.items()}


def iou_head_detector_config(variant: str = 'C1', num_reg_outs: int = 9) -> dict:
    """The synth detector config with FCAF3DHead and RotatedIoU3DLoss in place of FCAF3DHeadRotMat and BBoxCDLoss."""
    from embodiedscan_b200.synth import mv_det3d_config
    cfg = mv_det3d_config(variant)
    head = cfg['bbox_head']
    for k in ('decouple_bbox_loss', 'decouple_groups', 'decouple_weights'):
        head.pop(k)
    head.update(type='FCAF3DHead', num_reg_outs=num_reg_outs, bbox_loss=dict(type='RotatedIoU3DLoss', loss_weight=1.0))
    return cfg
