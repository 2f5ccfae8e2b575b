"""Distributed-evaluation cases shared by tests/test_eval_dist_cpu.py (gloo, oracle IoU) and tests/test_eval_dist_gpu.py
(the CUDA kernel): the golden metric fixtures split over W ranks the way mmengine's ``DefaultSampler(shuffle=False)``
splits a dataset, padding duplicates included, and the single-process result over the unpadded samples that every
rank's ``evaluate(size)`` must equal."""
import math
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
for p in (ROOT, HERE, os.path.join(HERE, 'golden')):
    if p not in sys.path:
        sys.path.insert(0, p)


def oracle_iou(p, q):
    from oracle import eval_ref as E
    return torch.from_numpy(E.iou_matrix(p.numpy(), q.numpy()))


def shard(n, world, rank):
    """DefaultSampler(shuffle=False): the index list padded by repetition to a multiple of `world`; rank r takes
    every W-th index from r."""
    total = math.ceil(n / world) * world
    idx = (list(range(n)) * (total // max(n, 1) + 1))[:total]
    return idx[rank:total:world]


def _det_units():
    from cases import eval_inputs
    gts, dts, metric, label2cat = eval_inputs()
    return [dict(eval_ann_info=g, pred_instances_3d=d) for g, d in zip(gts, dts)], metric, label2cat


def _det_prefixes(n_prefix):
    """Scan j (fixture scan j mod 4) as `n_prefix[j]` growing frame prefixes (the continuous configs' samples)."""
    samples, metric, label2cat = _det_units()
    units = []
    for j, c in enumerate(n_prefix):
        g, d = samples[j % len(samples)]['eval_ann_info'], samples[j % len(samples)]['pred_instances_3d']
        ng, nd = len(g['gt_labels_3d']), len(d['labels_3d'])
        unit = []
        for t in range(c):
            kg, kd = (ng * (t + 1)) // c, (nd * (t + 1)) // c
            ann = dict(gt_bboxes_3d=g['gt_bboxes_3d'][:kg], gt_labels_3d=g['gt_labels_3d'][:kg])
            unit.append(dict(eval_ann_info=ann, pred_instances_3d={k: v[:kd] for k, v in d.items()}))
        units.append(unit)
    return units, metric, label2cat


def _ground_units():
    from cases import grounding_metric_inputs
    dets, anns = grounding_metric_inputs()
    return [dict(eval_ann_info=a, pred_instances_3d=d) for d, a in zip(dets, anns)]


def _occ_units(device):
    from cases import occupancy_metric_inputs
    classes, samples = occupancy_metric_inputs()
    return [{k: v.to(device) for k, v in s.items()} for s in samples], classes


def cases(device='cpu', iou_fn=None):
    """name -> (metric factory, units, batch). A unit is one sample, or with batchwise_anns one scan's list of prefix
    samples (one `process` call); `batch` samples go to one `process` call otherwise."""
    from embodiedscan_b200.evaluation import GroundingMetric, IndoorDetMetric, OccupancyMetric
    det, metric, label2cat = _det_units()
    det_pre, _, _ = _det_prefixes([3, 1, 2, 4, 1])
    occ, classes = _occ_units(device)
    occ_pre = [[occ[(j + t) % 3] for t in range(c)] for j, c in enumerate([2, 1, 3, 1])]

    def det_metric(**kw):
        m = IndoorDetMetric(iou_thr=metric, iou_fn=iou_fn, **kw)
        m.dataset_meta = dict(classes=label2cat, classes_split=([2, 5], [9, 11], [40, 63, 77]))
        return m

    def occ_metric(**kw):
        m = OccupancyMetric(**kw)
        m.dataset_meta = dict(classes=classes)
        return m

    return {
        'det': (det_metric, det, 1),
        'det_batch2_prefix': (lambda: det_metric(prefix='val'), det, 2),
        'det_two_scans': (det_metric, det[:2], 1),
        'det_batchwise': (lambda: det_metric(batchwise_anns=True), det_pre, 1),
        'ground': (lambda: GroundingMetric(iou_thr=[0.25, 0.5], iou_fn=iou_fn), _ground_units(), 1),
        'ground_batch3_prefix': (lambda: GroundingMetric(iou_thr=[0.25, 0.5], iou_fn=iou_fn, prefix='test'),
                                 _ground_units(), 3),
        'occ': (occ_metric, occ, 1),
        'occ_one_scan': (occ_metric, occ[:1], 1),
        'occ_batchwise_prefix': (lambda: occ_metric(batchwise_anns=True, prefix='occ'), occ_pre, 1),
    }


def _feed(m, units, batch):
    if getattr(m, 'batchwise_anns', False):
        for unit in units:
            m.process(None, unit)
    else:
        for i in range(0, len(units), batch):
            m.process(None, units[i:i + batch])


def single_process(device='cpu', iou_fn=None):
    """Every case evaluated in one process over the unpadded samples in dataset order."""
    out = {}
    for name, (make, units, batch) in cases(device, iou_fn).items():
        m = make()
        _feed(m, units, batch)
        out[name] = m.evaluate()
    return out


def on_rank(rank, world, device='cpu', iou_fn=None):
    """Every case evaluated on this rank of an initialised process group, from the rank's DefaultSampler shard."""
    out = {}
    for name, (make, units, batch) in cases(device, iou_fn).items():
        m = make()
        _feed(m, [units[i] for i in shard(len(units), world, rank)], batch)
        out[name] = m.evaluate(size=len(units))
    return out


def first_difference(got, want):
    for name in want:
        if got[name] != want[name]:
            keys = sorted(set(got[name]) ^ set(want[name])) or \
                [k for k in want[name] if not (got[name][k] == want[name][k] or
                                               (np.isnan(got[name][k]) and np.isnan(want[name][k])))]
            return name, keys[:5]
    return None
