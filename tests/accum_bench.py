"""Time C2 bf16 training micro-batches (4 scans of 20 views 480x640 and 100k points each, fwd + loss + bwd through
`model.train_step`) with gradient accumulation over N = 1, 2 and 4 micro-batches per optimiser step, on one GPU. One model
and wrapper per N; rounds alternate the three so drift of the shared machine falls on all of them; each timed window is 8
micro-batches (whole windows for every N) between two device synchronisations, after 2 warm-up windows. Prints one JSON
object with the median and every round; DESIGN §6 quotes it.

On one GPU no micro-batch all-reduces, so what N changes here is the optimiser work per micro-batch (clip + AdamW +
bf16 shadow refresh + zero_grad once per N) and nothing else.

  python tests/accum_bench.py [--rounds 5] [--window 8]
"""
import argparse
import json
import os
import subprocess
import sys
import time

os.environ.setdefault('PYTORCH_CUDA_ALLOC_CONF', 'expandable_segments:True')      # as bench.py
import torch  # noqa: E402

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from embodiedscan_b200 import MODELS  # noqa: E402
from embodiedscan_b200.engine import OptimWrapper  # noqa: E402
from embodiedscan_b200.synth import mv_det3d_config, synth_scan  # noqa: E402

COUNTS = (1, 2, 4)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--rounds', type=int, default=5)
    ap.add_argument('--window', type=int, default=8, help='micro-batches per timed window (a multiple of every N)')
    args = ap.parse_args()
    assert torch.cuda.is_available(), 'accum_bench.py times the training step on a GPU'
    assert all(args.window % n == 0 for n in COUNTS)
    dev = torch.device('cuda', 0)
    batches = []
    for j in range(2):
        scans = [synth_scan(4 * j + i, augment=True, device=dev, n_views=20, H=480, W=640, n_points=100000)
                 for i in range(4)]
        batches.append(dict(inputs=dict(points=[s['points'] for s in scans], img=[s['img'] for s in scans]),
                            data_samples=[s['data_sample'] for s in scans]))
    runs = {}
    for n in COUNTS:
        torch.manual_seed(0)
        model = MODELS.build(dict(mv_det3d_config('C2'), compute_dtype=torch.bfloat16)).to(dev).train()
        runs[n] = (model, OptimWrapper(model, lr=1e-3, weight_decay=1e-4, max_norm=10.0, accumulative_counts=n))

    def window(n, count):
        model, ow = runs[n]
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        for j in range(count):
            model.train_step(batches[j % 2], ow)
        torch.cuda.synchronize()
        return time.perf_counter() - t0

    for n in COUNTS:
        window(n, 2 * args.window)
    times = {n: [] for n in COUNTS}
    for _ in range(args.rounds):
        for n in COUNTS:
            times[n].append(window(n, args.window))
    smi = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'],
                         capture_output=True, text=True).stdout.strip().splitlines()
    out = {'gpu': smi[0] if smi else torch.cuda.get_device_name(), 'micro_batch': 'C2: 4 scans x 20 views 480x640, 100k pts',
           'window_micro_batches': args.window, 'rounds': args.rounds}
    for n in COUNTS:
        ts = sorted(times[n])
        med = ts[len(ts) // 2]
        out[f'N={n}'] = {'micro_batches_per_s': args.window / med, 'ms_per_micro_batch': 1e3 * med / args.window,
                         'optimizer_steps': runs[n][1].optimizer.step_count,
                         'ms_per_micro_batch_rounds': [round(1e3 * t / args.window, 2) for t in times[n]]}
    print(json.dumps(out, indent=1))


if __name__ == '__main__':
    main()
