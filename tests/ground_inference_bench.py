"""Time grounding inference on one C4-shaped scan: 20 views 640x480 resized to 480x480, 100k points, the C4 grounder in
bf16 with the random-init text encoder (ESB200_TEXT_RANDOM_INIT=1; the RoBERTa weights do not change the work).

Routes, alternated in one process after a warm-up call of each:
* shared: ``inference_scan(prompts=K prompts)`` at K = 1, 12 and 48 (one visual pass, one decoder batch of K);
* per-sample: the reference's test loop at the config's batch size, K = 12 samples that each hold the scan and one
  prompt through ``data_preprocessor`` + ``predict`` (the visual branch runs for each), after the same scan-to-input
  step (depth unprojection, resize) that the shared route runs, done once.
Each time is a host clock around one call that ends in a device synchronise; the median and range over `--rounds`
rounds are reported as ms per call and per prompt, with the peak ``torch.cuda.max_memory_allocated`` of each route. The
K = 12 results of the two routes are compared query by query. The card's name and power limit are read in the same
process. Prints one JSON object; DESIGN §6 quotes it.

  python tests/ground_inference_bench.py [--rounds 5]
"""
import argparse
import json
import os
import subprocess
import sys
import time

os.environ.setdefault('ESB200_TEXT_RANDOM_INIT', '1')
os.environ.setdefault('PYTORCH_CUDA_ALLOC_CONF', 'expandable_segments:True')
HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, HERE)

import torch  # noqa: E402

from ground_inference_util import PROMPTS, grounder, predict_route  # noqa: E402

V, H, W, SCALE, N_POINTS, PER_VIEW = 20, 480, 640, (480, 480), 100000, 10000
SHARED_K = (1, 12, 48)
PER_SAMPLE_K = 12


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--rounds', type=int, default=5)
    args = ap.parse_args()
    assert torch.cuda.is_available(), 'ground_inference_bench.py times the GPU route'
    from embodiedscan_b200.inference import _scan_inputs, inference_scan
    from embodiedscan_b200.synth import synth_scan
    dev = torch.device('cuda', 0)
    model = grounder('C4', torch.bfloat16, dev)
    s = synth_scan(0, n_views=V, H=H, W=W, n_points=N_POINTS, device=dev)
    pm = s['data_sample'].metainfo['depth2img']
    scan = (s['img'].permute(0, 2, 3, 1).contiguous(), s['depth'], pm['intrinsic'][0], pm['extrinsic'])
    kw = dict(num_points=N_POINTS, points_per_view=PER_VIEW, seed=0, img_scale=SCALE)
    prompts = lambda k: [PROMPTS[i % len(PROMPTS)] for i in range(k)]

    def shared(k):
        return inference_scan(model, *scan, prompts=prompts(k), **kw)[0]

    def per_sample(k):
        points, img, meta = _scan_inputs(model, *scan, depth_shift=1000., **kw)
        return predict_route(model, points[0], img, meta, prompts(k))

    routes = {f'shared_K{k}': (shared, k) for k in SHARED_K}
    routes[f'per_sample_K{PER_SAMPLE_K}'] = (per_sample, PER_SAMPLE_K)
    outs = {name: fn(k) for name, (fn, k) in routes.items()}            # warm-up: every shape of the timed calls
    torch.cuda.synchronize()
    times = {name: [] for name in routes}
    peak = {name: 0 for name in routes}
    for _ in range(args.rounds):
        for name, (fn, k) in routes.items():
            torch.cuda.synchronize()
            torch.cuda.reset_peak_memory_stats(dev)
            t = time.perf_counter()
            fn(k)
            torch.cuda.synchronize()
            times[name].append(time.perf_counter() - t)
            peak[name] = max(peak[name], torch.cuda.max_memory_allocated(dev))
    res = {'workload': f'C4 grounder bf16, one scan: {V} views {W}x{H} -> {SCALE[0]}x{SCALE[1]}, {N_POINTS} points',
           'rounds': args.rounds}
    for name, (fn, k) in routes.items():
        t = sorted(times[name])
        res[name] = dict(ms_per_call=round(t[len(t) // 2] * 1e3, 1), ms_per_call_range=[round(t[0] * 1e3, 1),
                                                                                          round(t[-1] * 1e3, 1)],
                         ms_per_prompt=round(t[len(t) // 2] * 1e3 / k, 2), peak_alloc_GiB=round(peak[name] / 2 ** 30, 2))
    a, b = outs[f'shared_K{PER_SAMPLE_K}'], outs[f'per_sample_K{PER_SAMPLE_K}']
    sa = torch.stack([r.pred_instances_3d.scores_3d for r in a])
    sb = torch.stack([r.pred_instances_3d.scores_3d for r in b])
    ba = torch.stack([r.pred_instances_3d.bboxes_3d.tensor for r in a])
    bb = torch.stack([r.pred_instances_3d.bboxes_3d.tensor for r in b])
    res['K12_shared_vs_per_sample'] = dict(
        bit_identical=bool(torch.equal(sa, sb) and torch.equal(ba, bb)),
        max_rel_score_diff=float(((sa - sb).abs() / sb.abs()).max()),
        queries=int(sa.numel()),
        queries_with_a_box_off_by_over_0_01=int(((ba - bb).abs() > 1e-2).any(-1).sum()),
        same_top1_query=int(sum(int(x.argmax()) == int(y.argmax()) for x, y in zip(sa, sb))))
    res['speedup_K12'] = round(res[f'per_sample_K{PER_SAMPLE_K}']['ms_per_call'] / res['shared_K12']['ms_per_call'], 2)
    smi = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'],
                         capture_output=True, text=True).stdout.strip().splitlines()
    res['gpu'] = smi[0] if smi else torch.cuda.get_device_name()
    print(json.dumps(res, indent=1))


if __name__ == '__main__':
    main()
