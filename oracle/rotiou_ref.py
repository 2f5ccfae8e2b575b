"""Oracle (test infrastructure): the differentiable rotated 3D IoU of one-to-one box pairs in float64.

Restates mmcv.ops.diff_iou_rotated_3d (†upstream mmcv 2.0.0rc4, the IoU behind RotatedIoU3DLoss,
embodiedscan/models/losses/rotated_iou_loss.py:14-91) by its published algorithm; torch autograd gives the reference
gradients. Boxes are rows (x, y, z, w, l, h, alpha, ...) with z the box centre; columns past 7 are ignored.

  * BEV corners (+-w/2, +-l/2) in the order (+,+), (-,+), (-,-), (+,-), rotated counter-clockwise by alpha;
  * 24 candidate vertices: A's corners inside B, B's corners inside A, the 16 edge-edge intersections (index 4 i + j for
    A's edge i and B's edge j). Inside: the normalised projections on the two edges from corner 0 lie in
    (-1e-6, 1 + 1e-6). Intersections: strict 0 < t < 1 and 0 < u < 1; parallel edges give none;
  * the valid vertices sorted by angle about their mean (equal angles keep candidate order), the shoelace area of the
    cycle, 0 below 3 vertices. Gradients flow through the vertex coordinates, not through the order;
  * inter = area * clamp(min(top) - max(bottom), 0), iou = inter / (Va + Vb - inter), no epsilon. Ties of min / max and
    the clamp at 0 take torch autograd's rules.

No cap at 8 vertices: mmcv's CUDA vertex sort truncates there and rounds its own way; that stays parity unpinned.
"""
import torch

_SX = (0.5, -0.5, -0.5, 0.5)
_SY = (0.5, 0.5, -0.5, -0.5)


def bev_corners(boxes: torch.Tensor) -> torch.Tensor:
    """(N, >=7) -> (N, 4, 2)."""
    x, y, w, l, a = boxes[:, 0], boxes[:, 1], boxes[:, 3], boxes[:, 4], boxes[:, 6]
    px = boxes.new_tensor(_SX) * w[:, None]
    py = boxes.new_tensor(_SY) * l[:, None]
    c, s = torch.cos(a)[:, None], torch.sin(a)[:, None]
    return torch.stack((x[:, None] + px * c - py * s, y[:, None] + px * s + py * c), -1)


def _projections(p: torch.Tensor, q: torch.Tensor):
    """Normalised projections of points p (N, 4, 2) on the edges 0->1 and 0->3 of the rectangles q (N, 4, 2)."""
    a = q[:, 0:1]
    ab, ad, am = q[:, 1:2] - a, q[:, 3:4] - a, p - a
    return (ab * am).sum(-1) / (ab * ab).sum(-1), (ad * am).sum(-1) / (ad * ad).sum(-1)


def corners_inside(p: torch.Tensor, q: torch.Tensor) -> torch.Tensor:
    pab, pad = _projections(p, q)
    return (pab > -1e-6) & (pab < 1 + 1e-6) & (pad > -1e-6) & (pad < 1 + 1e-6)


def _edge_params(ca: torch.Tensor, cb: torch.Tensor):
    """(t, u, num, p1, p2) of every (A edge i, B edge j) pair, each (N, 4, 4[, 2])."""
    p1, p2 = ca[:, :, None, :], ca.roll(-1, 1)[:, :, None, :]
    p3, p4 = cb[:, None, :, :], cb.roll(-1, 1)[:, None, :, :]
    x1, y1, x2, y2 = p1[..., 0], p1[..., 1], p2[..., 0], p2[..., 1]
    x3, y3, x4, y4 = p3[..., 0], p3[..., 1], p4[..., 0], p4[..., 1]
    num = (x1 - x2) * (y3 - y4) - (y1 - y2) * (x3 - x4)
    safe = torch.where(num == 0, torch.ones_like(num), num)
    t = ((x1 - x3) * (y3 - y4) - (y1 - y3) * (x3 - x4)) / safe
    u = -((x1 - x2) * (y1 - y3) - (y1 - y2) * (x1 - x3)) / safe
    return t, u, num, p1, p2


def candidates(a: torch.Tensor, b: torch.Tensor):
    """The 24 candidate vertices (N, 24, 2) and their validity (N, 24)."""
    ca, cb = bev_corners(a), bev_corners(b)
    t, u, num, p1, p2 = _edge_params(ca, cb)
    ok = (num != 0) & (t > 0) & (t < 1) & (u > 0) & (u < 1)
    inter = p1 + t[..., None] * (p2 - p1)
    n = a.shape[0]
    verts = torch.cat((ca, cb, inter.reshape(n, 16, 2)), 1)
    valid = torch.cat((corners_inside(ca, cb), corners_inside(cb, ca), ok.reshape(n, 16)), 1)
    return verts, valid


def bev_intersection_area(a: torch.Tensor, b: torch.Tensor) -> torch.Tensor:
    verts, valid = candidates(a, b)
    n = valid.sum(1)
    with torch.no_grad():
        vf = valid.to(verts.dtype)[..., None]
        mean = (verts * vf).sum(1, keepdim=True) / n.clamp(min=1)[:, None, None].to(verts.dtype)
        d = verts - mean
        ang = torch.atan2(d[..., 1], d[..., 0]).masked_fill(~valid, float('inf'))
        order = torch.sort(ang, dim=1, stable=True).indices                 # valid first, by angle, ties by index
        k = torch.arange(24, device=verts.device).expand_as(order)
        nxt = torch.where(k + 1 < n[:, None], k + 1, torch.zeros_like(k))
        used = k < n[:, None]
    v = torch.gather(verts, 1, order[..., None].expand(-1, -1, 2))
    w = torch.gather(v, 1, nxt[..., None].expand(-1, -1, 2))
    s = ((v[..., 0] * w[..., 1] - v[..., 1] * w[..., 0]) * used).sum(1)
    return torch.where(n >= 3, s.abs() / 2, torch.zeros_like(s))


def diff_iou_rotated_3d(a: torch.Tensor, b: torch.Tensor) -> torch.Tensor:
    """One-to-one pairs a (N, >=7), b (N, >=7) -> iou (N,)."""
    area = bev_intersection_area(a, b)
    zmax = torch.min(a[:, 2] + a[:, 5] * 0.5, b[:, 2] + b[:, 5] * 0.5)
    zmin = torch.max(a[:, 2] - a[:, 5] * 0.5, b[:, 2] - b[:, 5] * 0.5)
    inter = area * (zmax - zmin).clamp(min=0.)
    va = a[:, 3] * a[:, 4] * a[:, 5]
    vb = b[:, 3] * b[:, 4] * b[:, 5]
    return inter / (va + vb - inter)


def iou_and_grads(a: torch.Tensor, b: torch.Tensor, grad_iou: torch.Tensor = None):
    """float64 iou (N,) and d sum(grad_iou * iou) / d a, b (N, 7)."""
    a = a[:, :7].detach().double().clone().requires_grad_(True)
    b = b[:, :7].detach().double().clone().requires_grad_(True)
    iou = diff_iou_rotated_3d(a, b)
    g = torch.ones_like(iou) if grad_iou is None else grad_iou.double()
    ga, gb = torch.autograd.grad(iou, (a, b), g)
    return iou.detach(), ga, gb


def degeneracy_margin(a: torch.Tensor, b: torch.Tensor) -> torch.Tensor:
    """float64 distance (metres) of each pair from the nearest configuration where a vertex enters or leaves the
    polygon or the z-overlap rule switches branch: corner-inside boundaries, intersection end points (t, u at 0 or 1,
    scaled by the edge lengths), the z overlap at 0 and ties of the tops / bottoms. fp32 and float64 may decide such a
    configuration differently, and the IoU's gradient is discontinuous there."""
    a, b = a[:, :7].double(), b[:, :7].double()
    ca, cb = bev_corners(a), bev_corners(b)
    m = []
    for p, q, box in ((ca, cb, b), (cb, ca, a)):
        pab, pad = _projections(p, q)
        for proj, size in ((pab, box[:, 3:4]), (pad, box[:, 4:5])):
            m.append(torch.minimum((proj + 1e-6).abs(), (proj - 1 - 1e-6).abs()) * size)
    t, u, num, _, _ = _edge_params(ca, cb)
    la = (ca.roll(-1, 1) - ca).norm(dim=-1)[:, :, None]
    lb = (cb.roll(-1, 1) - cb).norm(dim=-1)[:, None, :]
    par = num == 0
    big = torch.full_like(t, float('inf'))
    m.append(torch.where(par, big, torch.minimum(t.abs(), (1 - t).abs()) * la).flatten(1))
    m.append(torch.where(par, big, torch.minimum(u.abs(), (1 - u).abs()) * lb).flatten(1))
    at, ab_ = a[:, 2] + a[:, 5] / 2, a[:, 2] - a[:, 5] / 2
    bt, bb = b[:, 2] + b[:, 5] / 2, b[:, 2] - b[:, 5] / 2
    m.append(torch.stack(((torch.min(at, bt) - torch.max(ab_, bb)).abs(), (at - bt).abs(), (ab_ - bb).abs()), 1))
    return torch.cat([x.reshape(a.shape[0], -1) for x in m], 1).min(1).values
