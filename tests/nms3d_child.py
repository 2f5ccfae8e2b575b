"""Timing of the 3D-IoU box filter (csrc/nms3d.cu); pytest does not collect this file.

    python tests/nms3d_child.py --bench [--n 1000 4000 16000] [--iters 20]

Prints one JSON line per N. Candidates come from `nms3d_ref.cluster_boxes`: N / 10 cuboids at 24 per 6 m x 6 m of floor
(the density of a synth room; the floor grows with N), each with 10 jittered copies (centre sigma 8 cm, log-size sigma
0.12, angles sigma 0.12 rad), 20 labels, uniform scores. This cluster model decides how many pairs survive the early
rejects, so the counts are reported with the times: pairs tested, pairs left by the bounding-sphere test, pairs left by
the separating-axis test (those run the exact clipping).

  nms3d_ms        esb_nms3d_9dof (both kernels, sorted input on the device), CUDA events, median
  pair_ms/greedy_ms  the two kernels of that call, from torch.profiler in a pass of its own
  matrix_route_ms the route without this kernel: esb_box3d_overlap full N x N matrix, threshold on the device, copy to the
                  host, greedy walk in numpy; host clock around work that ends synchronised, median of fewer repeats
The two routes alternate in the same process; their kept lists are compared. Filter: iou 0.15, score 0.075, 10 per label."""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

IOU_THR, SCORE_THR, TOPK, NUM_CLASSES = 0.15, 0.075, 10, 20


def _power_limit_w():
    try:
        out = subprocess.run(['nvidia-smi', '--query-gpu=power.limit', '--format=csv,noheader,nounits', '-i',
                              str(torch.cuda.current_device())], capture_output=True, text=True, timeout=30)
        return float(out.stdout.strip().splitlines()[0])
    except Exception:
        return None


def _median(v):
    v = sorted(v)
    return v[len(v) // 2]


def bench(N, iters):
    from embodiedscan_b200 import _ffi
    from embodiedscan_b200.geometry import box3d_overlap, box_corners_container
    from nms3d_ref import cluster_boxes
    assert torch.cuda.is_available(), 'the timing needs a GPU'
    boxes, scores, labels = cluster_boxes(N, 0, copies=10, per_room=24, num_classes=NUM_CLASSES)[:3]
    order = np.argsort(-scores, kind='stable')
    b = torch.from_numpy(boxes[order]).cuda().contiguous()
    sc = torch.from_numpy(scores[order]).cuda().contiguous()
    lab = torch.from_numpy(labels[order].astype(np.int32)).cuda().contiguous()
    lab_host = labels[order]
    so = torch.tensor([0, N], dtype=torch.int32, device='cuda')
    keep = torch.empty(N, dtype=torch.int32, device='cuda')
    n_keep = torch.zeros(1, dtype=torch.int32, device='cuda')
    wsb = _ffi.query('esb_nms3d_9dof_workspace_bytes', N, 1, N)
    ws = torch.empty(wsb, dtype=torch.uint8, device='cuda')

    def ours():
        _ffi.call('esb_nms3d_9dof', b.data_ptr(), sc.data_ptr(), lab.data_ptr(), so.data_ptr(), 1, N, IOU_THR, SCORE_THR,
                  TOPK, NUM_CLASSES, keep.data_ptr(), n_keep.data_ptr(), ws.data_ptr(), wsb, _ffi.stream())

    def matrix_route():
        k = box_corners_container(b)
        over = (box3d_overlap(k, k)[1] > IOU_THR).cpu().numpy()               # over[i][j]: candidate i against kept j
        ok = (sc >= SCORE_THR).cpu().numpy()
        selected, per_label = [], {}
        for i in range(N):
            if per_label.get(lab_host[i], 0) >= TOPK or not ok[i]:
                continue
            if selected and over[i, selected].any():
                continue
            selected.append(i)
            per_label[lab_host[i]] = per_label.get(lab_host[i], 0) + 1
        return selected

    ours()
    ref_keep = matrix_route()
    torch.cuda.synchronize()
    mine = keep[:int(n_keep.item())].tolist()
    stats = ws[:24].view(torch.int64).tolist()
    start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    t_ours, t_route = [], []
    route_every = max(1, iters // 3)
    for it in range(iters):                                                   # the two routes alternate
        start.record()
        ours()
        end.record()
        torch.cuda.synchronize()
        t_ours.append(start.elapsed_time(end))
        if it % route_every == 0:
            t0 = time.perf_counter()
            matrix_route()
            torch.cuda.synchronize()
            t_route.append((time.perf_counter() - t0) * 1e3)
    pair_ms = greedy_ms = None
    try:
        from torch.profiler import ProfilerActivity, profile
        reps = 5
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(reps):
                ours()
            torch.cuda.synchronize()
        for ev in prof.key_averages():
            total = getattr(ev, 'device_time_total', None)
            total = getattr(ev, 'cuda_time_total', 0.0) if total is None else total
            if 'nms3d_pair_kernel' in ev.key:
                pair_ms = round(total / reps / 1e3, 4)
            elif 'nms3d_greedy_kernel' in ev.key:
                greedy_ms = round(total / reps / 1e3, 4)
    except Exception as e:                                                    # the split is extra; the totals stand
        print(f'profiler pass failed: {e}', file=sys.stderr)
    print(json.dumps(dict(N=N, kept=len(mine), same_keep_as_matrix_route=mine == ref_keep, pairs_tested=stats[0],
                          pairs_past_sphere=stats[1], pairs_past_sat=stats[2], nms3d_ms=round(_median(t_ours), 4),
                          pair_ms=pair_ms, greedy_ms=greedy_ms, matrix_route_ms=round(_median(t_route), 2),
                          matrix_route_repeats=len(t_route), iters=iters, mask_bytes=wsb,
                          card=torch.cuda.get_device_name(), power_limit_w=_power_limit_w())), flush=True)


if __name__ == '__main__':
    ap = argparse.ArgumentParser()
    ap.add_argument('--bench', action='store_true')
    ap.add_argument('--n', type=int, nargs='+', default=[1000, 4000, 16000])
    ap.add_argument('--iters', type=int, default=20)
    a = ap.parse_args()
    if a.bench:
        for n in a.n:
            bench(n, a.iters)
