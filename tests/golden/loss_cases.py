"""Seeded inputs of the chamfer-loss fixture (tests/golden/losses.npz, written by make_golden_losses.py).

Outside deliberate exact duplicates, every point set keeps a relative margin of at least MARGIN between the best and the
second-best candidate of every nearest-neighbour search, so fp32 rounding cannot flip an arg-minimum."""
import torch

MARGIN = 1e-4
MODES = ('l1', 'l2', 'smooth_l1')
REDUCTIONS = ('mean', 'sum', 'none')
GROUPS = ('g8', 'g4')


def criterion_distance(a, b, mode):
    """(..., N, C), (..., M, C) -> (..., N, M): the criterion summed over coordinates, in float64."""
    x = a.double()[..., :, None, :] - b.double()[..., None, :, :]
    if mode == 'l1':
        return x.abs().sum(-1)
    if mode == 'l2':
        return (x * x).sum(-1)
    ax = x.abs()
    return torch.where(ax < 1, 0.5 * ax * ax, ax - 0.5).sum(-1)


def relative_margin(d):
    """min over rows of (second best - best) / max(best, 1e-6) along the last dim of d (rows with one candidate: inf)."""
    if d.shape[-1] < 2:
        return float('inf')
    top = d.topk(2, dim=-1, largest=False).values
    return float(((top[..., 1] - top[..., 0]) / top[..., 0].clamp(min=1e-6)).min())


def set_margin(src, dst):
    """Smallest relative margin of both search directions over every criterion."""
    return min(min(relative_margin(criterion_distance(src, dst, m)), relative_margin(criterion_distance(dst, src, m)))
               for m in MODES)


def _points(g, B, N, C, scale):
    return (torch.rand(B, N, C, generator=g) * 2 - 1) * scale


def chamfer_cases():
    """name -> dict(src (B,N,C), dst (B,M,C), src_weight, dst_weight); weights are floats or positive tensors."""
    g = torch.Generator().manual_seed(101)
    cases = {}

    def draw(B, N, M, C, scale):
        while True:
            src, dst = _points(g, B, N, C, scale), _points(g, B, M, C, scale)
            if set_margin(src, dst) >= MARGIN:
                return src, dst

    src, dst = draw(2, 37, 53, 3, 1.5)             # spans both smooth-L1 branches
    cases['c3_float'] = dict(src=src, dst=dst, src_weight=0.7, dst_weight=1.3)
    src, dst = draw(3, 20, 11, 2, 0.8)
    cases['c2_tensor'] = dict(src=src, dst=dst, src_weight=0.5 + torch.rand(3, 20, generator=g),
                              dst_weight=0.5 + torch.rand(3, 11, generator=g))
    src, dst = draw(2, 1, 9, 3, 1.0)
    cases['n1'] = dict(src=src, dst=dst, src_weight=1.0, dst_weight=1.0)
    # exact duplicates in both sets: the first of two equal candidates must win
    while True:
        src, dst = _points(g, 1, 12, 3, 1.0), _points(g, 1, 10, 3, 1.0)
        if set_margin(src, dst) >= MARGIN:
            break
    src[0, 9] = src[0, 2]
    dst[0, 7] = dst[0, 3]
    src[0, 5] = dst[0, 3]          # a source point on a duplicated target point: distance 0 to both copies
    cases['duplicates'] = dict(src=src, dst=dst, src_weight=1.0, dst_weight=1.0)
    return cases


def _boxes(g, n, dim):
    ctr = torch.rand(n, 3, generator=g) * 4 - 2
    size = 0.3 + torch.rand(n, 3, generator=g) * 1.5
    ang = torch.stack([torch.rand(n, generator=g) * 6 - 3, 0.3 * torch.randn(n, generator=g),
                       0.3 * torch.randn(n, generator=g)], 1)
    return torch.cat([ctr, size, ang], 1)[:, :dim]


def bbox_cases(corners_of):
    """dim -> (source (N,dim), target (N,dim), weight): sources are jittered targets. `corners_of` maps boxes to
    (N, 8, 3) corners; pairs are redrawn until both corner groups keep the margin."""
    g = torch.Generator().manual_seed(202)
    out = {}
    for dim, weight in ((6, 0.8), (7, 'tensor'), (9, 1.0)):
        n = 10
        while True:
            tgt = _boxes(g, n, dim)
            src = tgt + 0.25 * torch.randn(n, dim, generator=g)
            src[:, 3:6] = src[:, 3:6].abs() + 0.1
            sc, tc = corners_of(src), corners_of(tgt)
            ok = all(relative_margin(criterion_distance(sc, tc, m)) >= MARGIN and
                     relative_margin(criterion_distance(sc[:, :4], tc[:, :4], m)) >= MARGIN and
                     relative_margin(criterion_distance(sc[:, 4:], tc[:, 4:], m)) >= MARGIN for m in MODES)
            if ok:
                break
        w = 0.5 + torch.rand(n, 1, generator=g) if weight == 'tensor' else weight
        out[dim] = (src, tgt, w)
    return out


def head_loss_inputs(target_cases):
    """Two scans for FCAF3DHeadRotMat.loss_by_feat: per level, per scan points / centre / 12-channel box / class
    predictions. Scan 0 holds the 'regular' target case, scan 1 the 'few_points' case."""
    g = torch.Generator().manual_seed(303)
    tc = target_cases()
    scans = [tc['regular'], tc['few_points']]
    points = [[scans[b][0][l].clone() for b in range(2)] for l in range(4)]
    center, bbox, cls = [], [], []
    for l in range(4):
        center.append([torch.randn(len(points[l][b]), 1, generator=g) for b in range(2)])
        bbox.append([torch.cat([0.2 + torch.rand(len(points[l][b]), 6, generator=g),
                                torch.randn(len(points[l][b]), 6, generator=g)], 1) for b in range(2)])
        cls.append([torch.randn(len(points[l][b]), 284, generator=g) - 3 for b in range(2)])
    gts = [(scans[b][1], scans[b][2]) for b in range(2)]
    return points, center, bbox, cls, gts


HEAD_GRID = [(mode, group, norm, dec) for mode in MODES for group in GROUPS for norm in (False, True)
             for dec in (0, 3, 4)]


def head_config_name(mode, group, norm, dec):
    return f'{mode}_{group}_{"norm" if norm else "plain"}_d{dec}'
