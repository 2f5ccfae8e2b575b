"""esb_box3d_best_overlap against the full box3d_overlap matrix: on seeded clustered scans (thin predictions after the
2e-4 clamp, identical and duplicated boxes, zero-size ground truth, scans without same-class ground truth, empty scans,
284 labels) and on the grounding layout (top-10 candidates x a prompt's targets), `best` and `arg` are bit-identical to
the matrix masked to the query's range and reduced on the host by torch.max (first maximum; a NaN wins)."""
import os
import sys

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu
DEV = 'cuda:0'


def _host_best(iou, mask):
    """today's host rule: mask to the range, first maximum, -inf / -1 where the range is empty"""
    b, a = torch.where(mask, iou, torch.full_like(iou, -1.0)).max(dim=1)
    has = mask.any(1)
    return torch.where(has, b, torch.full_like(b, float('-inf'))), torch.where(has, a, torch.full_like(a, -1))


def _check(cq, ct, tidx, qbeg, qend, mask):
    from embodiedscan_b200.geometry import box3d_best_overlap, box3d_overlap
    best, arg = box3d_best_overlap(cq, ct, tidx, qbeg, qend)
    torch.cuda.synchronize()
    want_b, want_a = _host_best(box3d_overlap(cq, ct)[1].cpu(), mask)
    assert torch.equal(best.cpu().view(torch.int32), want_b.view(torch.int32)), \
        int((best.cpu().view(torch.int32) != want_b.view(torch.int32)).sum())
    assert torch.equal(arg.cpu().long(), want_a)
    return best.cpu(), want_a


def _clustered_scans(g, n_scans=48):
    """Per scan: GT in a few clusters (some zero-size, some duplicated), predictions = jittered / identical / thin
    copies with the GT's label or a random one, plus noise. Some scans have no GT, no predictions, or no shared
    label."""
    scans = []
    for s in range(n_scans):
        n_gt = [0, 1, 7, 60][s % 4] if s % 11 else 0
        n_pred = [300, 0, 40, 1000][s % 4] if s % 13 else 0
        ctr = torch.rand(max(n_gt, 1) // 6 + 1, 3, generator=g) * 6
        at = ctr[torch.randint(0, ctr.shape[0], (n_gt, ), generator=g)] + 0.4 * torch.randn(n_gt, 3, generator=g)
        gb = torch.cat([at, 0.2 + torch.rand(n_gt, 3, generator=g), 0.3 * torch.randn(n_gt, 3, generator=g)], 1)
        gl = torch.randint(0, 284, (n_gt, ), generator=g)
        if n_gt >= 7:
            gl[:n_gt // 2] = gl[0]                               # many boxes of one label: long ranges
            gb[1, 3:6] = 0.0                                     # zero-size ground truth
            gb[2, 4] = 0.0
            gb[3], gl[3] = gb[4], gl[4]                          # duplicated box: a tie, the smaller index wins
        src = torch.randint(0, max(n_gt, 1), (n_pred, ), generator=g)
        pb = 6 * torch.rand(n_pred, 9, generator=g)
        pl = torch.randint(0, 284, (n_pred, ), generator=g)
        if n_gt:
            mag = torch.tensor([0., 0.02, 0.1, 0.3])[torch.randint(0, 4, (n_pred, ), generator=g)][:, None]
            pb = gb[src] + mag * torch.randn(n_pred, 9, generator=g)
            same = torch.rand(n_pred, generator=g) < 0.8
            pl = torch.where(same, gl[src], pl)
            thin = torch.rand(n_pred, generator=g) < 0.05
            pb[thin, 4] = 1e-4                                   # face areas below 2e-4: clamped to 2e-2 edges
            pb[:, 3:6] = pb[:, 3:6].abs()
        if s % 7 == 3:
            pl = (gl.max() + 1 if n_gt else 0) + pl % 3          # no same-class ground truth in this scan
        scans.append((pb, pl, gb, gl))
    return scans


def test_detection_layout_bit_identical_to_the_masked_matrix():
    from embodiedscan_b200.evaluation import _clamp_thin, _corners, same_class_ranges
    g = torch.Generator().manual_seed(2024)
    scans = _clustered_scans(g)
    pscan = torch.cat([torch.full((sc[0].shape[0], ), i) for i, sc in enumerate(scans)])
    gscan = torch.cat([torch.full((sc[2].shape[0], ), i) for i, sc in enumerate(scans)])
    pl, gl = torch.cat([sc[1] for sc in scans]), torch.cat([sc[3] for sc in scans])
    pb = _clamp_thin(torch.cat([sc[0] for sc in scans]))
    gb = torch.cat([sc[2] for sc in scans])
    dev = torch.device(DEV)
    cq, ct = _corners(pb, dev), _corners(gb, dev)
    tidx, qbeg, qend = same_class_ranges(pscan.to(dev), pl.to(dev), gscan.to(dev), gl.to(dev))
    mask = (pscan[:, None] == gscan[None]) & (pl[:, None] == gl[None])
    assert torch.equal((qend - qbeg).cpu(), mask.sum(1))
    best, arg = _check(cq, ct, tidx, qbeg, qend, mask)
    assert len(set(pl.tolist() + gl.tolist())) > 250
    hit = arg >= 0
    assert 0 < int(hit.sum()) < best.numel()                                 # both matched and unmatched queries
    assert bool((best[hit] > 0.999).any())                                   # identical boxes
    assert int((qend - qbeg).max()) >= 20


def test_degenerate_boxes_pick_what_torch_max_picks():
    """inf / NaN coordinates and sizes, all-zero boxes: whatever the pair routine yields (NaN included), the reduction
    is torch.max's."""
    g = torch.Generator().manual_seed(7)
    n = 64
    gb = torch.cat([torch.rand(n, 3, generator=g), 0.5 + torch.rand(n, 3, generator=g), torch.zeros(n, 3)], 1)
    pb = gb[torch.randint(0, n, (n, ), generator=g)] + 0.05 * torch.randn(n, 9, generator=g)
    bad = torch.tensor([float('inf'), float('nan'), -float('inf'), 0.0, 1e30])
    for k in range(0, n, 3):
        pb[k, k % 9] = bad[k % 5]
        gb[(k + 1) % n, (k + 4) % 9] = bad[(k + 2) % 5]
    dev = torch.device(DEV)
    from embodiedscan_b200.evaluation import _corners
    cq, ct = _corners(pb, dev), _corners(gb, dev)
    qbeg = torch.randint(0, n, (n, ), generator=g)
    qend = torch.minimum(qbeg + torch.randint(0, 12, (n, ), generator=g), torch.tensor(n))
    mask = (torch.arange(n)[None] >= qbeg[:, None]) & (torch.arange(n)[None] < qend[:, None])
    _check(cq, ct, torch.arange(n), qbeg, qend, mask)


def test_grounding_layout_bit_identical_to_the_masked_matrix():
    """one query per top-10 candidate, its range = the targets of its prompt (0 to 3 of them)"""
    g = torch.Generator().manual_seed(99)
    prompts = 37
    nc = torch.randint(0, 11, (prompts, ), generator=g)
    nt = torch.randint(0, 4, (prompts, ), generator=g)
    tb = torch.cat([2 * torch.rand(int(nt.sum()), 3, generator=g), 0.3 + torch.rand(int(nt.sum()), 3, generator=g),
                    0.3 * torch.randn(int(nt.sum()), 3, generator=g)], 1)
    tprompt = torch.repeat_interleave(torch.arange(prompts), nt)
    cprompt = torch.repeat_interleave(torch.arange(prompts), nc)
    toff = torch.cumsum(nt, 0) - nt
    pick = [int(toff[p]) + int(torch.randint(0, max(int(nt[p]), 1), (1, ), generator=g)) for p in cprompt.tolist()]
    cb = torch.cat([2 * torch.rand(int(nc.sum()), 3, generator=g), 0.3 + torch.rand(int(nc.sum()), 3, generator=g),
                    0.3 * torch.randn(int(nc.sum()), 3, generator=g)], 1)
    near = torch.tensor([nt[p] > 0 for p in cprompt.tolist()]) & (torch.rand(int(nc.sum()), generator=g) < 0.5)
    cb[near] = tb[torch.tensor(pick)[near]] + 0.1 * torch.randn(int(near.sum()), 9, generator=g)
    cb[:, 3:6] = cb[:, 3:6].abs()
    dev = torch.device(DEV)
    from embodiedscan_b200.evaluation import _corners
    qbeg = torch.repeat_interleave(toff, nc)
    qend = qbeg + torch.repeat_interleave(nt, nc)
    best, _ = _check(_corners(cb, dev), _corners(tb, dev), torch.arange(tb.shape[0]), qbeg, qend,
                     cprompt[:, None] == tprompt[None])
    assert bool((best > 0.25).any()) and bool((best == float('-inf')).any())


def _per_scan_matrix(pred9, gt9):
    """the route indoor_eval and GroundingMetric took before: one full esb_box3d_overlap matrix per scan / prompt"""
    from embodiedscan_b200.evaluation import _corners
    from embodiedscan_b200.geometry import box3d_overlap
    return box3d_overlap(_corners(pred9, torch.device(DEV)), _corners(gt9, torch.device(DEV)))[1]


def test_records_and_grounding_hits_equal_the_per_scan_matrix_route_bit_for_bit():
    """Stage (a) of indoor_eval hands stage (b) the arrays the per-scan matrix route gave it, bit for bit, and the
    grounding hits are the same, on the golden fixtures and on the clustered scans."""
    from embodiedscan_b200.evaluation import GroundingMetric, detection_records
    sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden'))
    from cases import eval_inputs, grounding_metric_inputs
    gts, dts, _, _ = eval_inputs()
    scans = _clustered_scans(torch.Generator().manual_seed(5), n_scans=30)
    gts += [dict(gt_bboxes_3d=gb.numpy(), gt_labels_3d=gl.numpy()) for _, _, gb, gl in scans]
    dts += [dict(bboxes_3d=pb.numpy(), labels_3d=pl.numpy(), scores_3d=np.linspace(0, 1, len(pl), dtype=np.float32))
            for pb, pl, _, _ in scans]
    new, old = detection_records(gts, dts), detection_records(gts, dts, _per_scan_matrix)
    for f, x, y in zip(new._fields, new, old):
        assert x.dtype == y.dtype and np.array_equal(x.view(np.uint8), y.view(np.uint8)), f
    assert int((new.best > 0.5).sum()) > 100
    dets, anns = grounding_metric_inputs()
    m = GroundingMetric(iou_thr=[0.25, 0.5])
    assert torch.equal(m._found(anns, dets, None), m._found(anns, dets, _per_scan_matrix))
