"""Time ``indoor_eval`` at user scale: the same-class matching in one ``esb_box3d_best_overlap`` launch (this library)
against the route it replaced, written out here: per scan the full predictions x ground-truth matrix from
``esb_box3d_overlap``, copied to the host and masked to equal labels there.

    python tests/eval_bench.py [--scans 300 --preds 1000 --gts 60 --rounds 5]

A seeded synthetic set: per scan, ground-truth boxes in clusters over 284 labels; predictions are jittered copies of
them (mostly with the box's label) and random boxes with random labels. Both routes run in one process, alternating,
after one warm-up call each, with a host clock around work that ends synchronised. The two result dicts must be equal,
and so must the per-detection records, bit for bit.
Prints one JSON line with the card's name and power limit, the pairs each route clips and the times."""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from embodiedscan_b200 import evaluation as E  # noqa: E402
from embodiedscan_b200.geometry import box3d_overlap  # noqa: E402


def synthetic(n_scans, n_pred, n_gt, n_labels=284, seed=0):
    g = np.random.default_rng(seed)
    gts, dts = [], []
    for _ in range(n_scans):
        ctr = g.uniform([0, 0, 0], [8, 8, 2.5], (n_gt // 6 + 1, 3))[g.integers(0, n_gt // 6 + 1, n_gt)]
        gb = np.concatenate([ctr + g.normal(0, 0.6, (n_gt, 3)), g.uniform(0.2, 1.5, (n_gt, 3)),
                             g.normal(0, 0.3, (n_gt, 3))], 1).astype(np.float32)
        gl = g.integers(0, n_labels, n_gt)
        n_copy = int(0.6 * n_pred)
        src = g.integers(0, n_gt, n_copy)
        pc = gb[src] + g.normal(0, 1, (n_copy, 9)).astype(np.float32) * g.choice([0.02, 0.1, 0.3], (n_copy, 1))
        pc[:, 3:6] = np.abs(pc[:, 3:6])
        pr = np.concatenate([g.uniform([0, 0, 0], [8, 8, 2.5], (n_pred - n_copy, 3)),
                             g.uniform(0.1, 1.5, (n_pred - n_copy, 3)), g.normal(0, 0.3, (n_pred - n_copy, 3))], 1)
        pl = np.concatenate([np.where(g.random(n_copy) < 0.85, gl[src], g.integers(0, n_labels, n_copy)),
                             g.integers(0, n_labels, n_pred - n_copy)])
        gts.append(dict(gt_bboxes_3d=gb, gt_labels_3d=gl))
        dts.append(dict(bboxes_3d=np.concatenate([pc, pr]).astype(np.float32), labels_3d=pl,
                        scores_3d=g.random(n_pred).astype(np.float32)))
    return gts, dts


def previous_iou(pred9, gt9):
    """the replaced route's IoU: the full matrix of one scan on the device, copied to the host (masked by the caller)"""
    dev = torch.device('cuda', torch.cuda.current_device())
    return box3d_overlap(E._corners(pred9, dev), E._corners(gt9, dev))[1].cpu()


def timed(fn):
    torch.cuda.synchronize()
    t = time.perf_counter()
    out = fn()
    torch.cuda.synchronize()
    return time.perf_counter() - t, out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--scans', type=int, default=300)
    ap.add_argument('--preds', type=int, default=1000)
    ap.add_argument('--gts', type=int, default=60)
    ap.add_argument('--rounds', type=int, default=5)
    a = ap.parse_args()
    assert torch.cuda.is_available(), 'eval_bench times the GPU: a CUDA device is required'
    smi = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader', '-i', '0'],
                         capture_output=True, text=True).stdout.strip()
    gts, dts = synthetic(a.scans, a.preds, a.gts)
    label2cat = {i: f'class{i}' for i in range(284)}
    thr = [0.25, 0.5]
    routes = {'best_overlap': lambda: E.indoor_eval(gts, dts, thr, label2cat),
              'full_matrix': lambda: E.indoor_eval(gts, dts, thr, label2cat, iou_fn=previous_iou)}
    stage_a = {'best_overlap': lambda: E.detection_records(gts, dts),
               'full_matrix': lambda: E.detection_records(gts, dts, previous_iou)}
    results = {k: fn() for k, fn in routes.items()}                  # warm-up
    assert results['best_overlap'] == results['full_matrix'], 'the two routes disagree'
    for fn in stage_a.values():
        fn()
    times = {k: [] for k in routes}
    times_a = {k: [] for k in routes}
    for _ in range(a.rounds):
        for k in routes:
            dt, out = timed(routes[k])
            assert out == results[k]
            times[k].append(dt)
            times_a[k].append(timed(stage_a[k])[0])
    rec_new, rec_old = stage_a['best_overlap'](), stage_a['full_matrix']()
    for f, x, y in zip(rec_new._fields, rec_new, rec_old):         # every record, bit for bit
        assert x.dtype == y.dtype and np.array_equal(x.view(np.uint8), y.view(np.uint8)), f
    pairs_full = sum(len(d['labels_3d']) * len(g['gt_labels_3d']) for g, d in zip(gts, dts))
    pairs_same = sum(int((np.asarray(d['labels_3d'])[:, None] == np.asarray(g['gt_labels_3d'])[None]).sum())
                     for g, d in zip(gts, dts))
    ms = (lambda xs: [round(1e3 * x, 2) for x in xs])
    print(json.dumps({
        'gpu': smi, 'scans': a.scans, 'preds_per_scan': a.preds, 'gts_per_scan': a.gts, 'labels': 284,
        'pairs_clipped': {'best_overlap': pairs_same, 'full_matrix': pairs_full},
        'indoor_eval_ms': {k: ms(v) for k, v in times.items()},
        'indoor_eval_ms_median': {k: round(1e3 * statistics.median(v), 2) for k, v in times.items()},
        'matching_stage_ms': {k: ms(v) for k, v in times_a.items()},
        'matching_stage_ms_median': {k: round(1e3 * statistics.median(v), 2) for k, v in times_a.items()},
        'mAP_0.25': results['best_overlap']['mAP_0.25'], 'results_equal': True, 'records_bit_identical': True}))


if __name__ == '__main__':
    main()
