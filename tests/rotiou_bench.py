"""Timing of the rotated 3D IoU kernel (csrc/rotiou3d.cu) and of the detector step with FCAF3DHead; pytest does not
collect this file.

    python tests/rotiou_bench.py [--pairs 4096 32768 262144] [--iters 50] [--steps 5] [--rounds 3] [--no-step]

Prints one JSON line per measurement, each with the card's name and power limit read in the same process.

  kernel_ms  esb_rotated_iou3d_fwd + esb_rotated_iou3d_bwd through rotated_iou_3d and autograd, for P pairs; median over
             rounds of CUDA-event windows of `iters` calls after warm-up
  aten_ms    the same forward + backward of the fp32 ATen restatement (oracle/rotiou_ref.py run on the GPU in fp32),
             alternated with the kernel in the same process
  step_ms    one C2-shaped bf16 training step (4 scans, 20 views of 480 x 640, 100k points, synth inputs) of the detector
             with FCAF3DHead (9 outputs, RotatedIoU3DLoss) against the same detector with FCAF3DHeadRotMat (the C2
             config), alternating windows of `steps` steps; median per-step time over rounds
Pairs are the seeded population of rotiou_util.random_pairs (4096 drawn pairs, repeated and jittered by 1 cm)."""
import argparse
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))


def card():
    try:
        out = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader', '-i',
                              str(torch.cuda.current_device())], capture_output=True, text=True, timeout=30)
        name, power = [s.strip() for s in out.stdout.strip().splitlines()[0].split(',')]
        return dict(card=name, power_limit=power)
    except Exception as e:                       # the numbers still print; the card is then unknown
        return dict(card=torch.cuda.get_device_name(), power_limit=f'unknown ({e})')


def _median(v):
    v = sorted(v)
    return v[len(v) // 2]


def _window(fn, iters):
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    s.record()
    for _ in range(iters):
        fn()
    e.record()
    torch.cuda.synchronize()
    return s.elapsed_time(e) / iters


def bench_kernel(P, iters, rounds, meta):
    from embodiedscan_b200 import rotated_iou_3d
    from oracle import rotiou_ref as R
    from rotiou_util import random_pairs
    a0, b0 = random_pairs(4096, 0)
    rep = (P + 4095) // 4096
    a = a0.repeat(rep, 1)[:P].cuda()
    b = b0.repeat(rep, 1)[:P].cuda()
    a += torch.randn(a.shape, generator=torch.Generator().manual_seed(1)).cuda() * 0.01
    g = torch.ones(P, device='cuda')
    a.requires_grad_(True)
    b.requires_grad_(True)

    def ours():
        torch.autograd.grad(rotated_iou_3d(a, b), (a, b), g)

    def aten():
        torch.autograd.grad(R.diff_iou_rotated_3d(a, b), (a, b), g)

    with torch.no_grad():
        ref = R.diff_iou_rotated_3d(a.double(), b.double())
        err = float((rotated_iou_3d(a, b).double() - ref).abs().max())
    for f in (ours, aten):
        for _ in range(3):
            f()
    torch.cuda.synchronize()
    t_ours, t_aten = [], []
    for _ in range(rounds):
        t_ours.append(_window(ours, iters))
        t_aten.append(_window(aten, max(1, iters // 5)))
    print(json.dumps(dict(meta, what='rotated_iou3d fwd+bwd', pairs=P, kernel_ms=round(_median(t_ours), 4),
                          aten_ms=round(_median(t_aten), 4), kernel_rounds=[round(t, 4) for t in t_ours],
                          aten_rounds=[round(t, 4) for t in t_aten], max_abs_iou_err_vs_fp64=err)), flush=True)


def bench_step(steps, rounds, meta):
    from embodiedscan_b200 import MODELS
    from embodiedscan_b200.engine import OptimWrapper
    from embodiedscan_b200.synth import mv_det3d_config, synth_scan
    from rotiou_util import iou_head_detector_config
    scans = [synth_scan(i, augment=True, device='cuda', n_views=20, H=480, W=640, n_points=100000) for i in range(4)]
    data = dict(inputs=dict(points=[s['points'] for s in scans], img=[s['img'] for s in scans]),
                data_samples=[s['data_sample'] for s in scans])
    runs = {}
    for name, cfg in (('FCAF3DHead', iou_head_detector_config('C2', 9)), ('FCAF3DHeadRotMat', mv_det3d_config('C2'))):
        torch.manual_seed(0)
        model = MODELS.build(dict(cfg, compute_dtype=torch.bfloat16)).cuda().train()
        optim = OptimWrapper(model, lr=1e-3, weight_decay=1e-4, max_norm=10.0)
        runs[name] = (model, optim)
        for _ in range(3):
            model.train_step(data, optim)
    torch.cuda.synchronize()
    times = {k: [] for k in runs}
    for _ in range(rounds):
        for name, (model, optim) in runs.items():
            times[name].append(_window(lambda: model.train_step(data, optim), steps))
    print(json.dumps(dict(meta, what='C2-shaped bf16 training step', **{f'{k}_step_ms': round(_median(v), 2)
                                                                        for k, v in times.items()},
                          rounds={k: [round(t, 2) for t in v] for k, v in times.items()})), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--pairs', type=int, nargs='+', default=[4096, 32768, 262144])
    ap.add_argument('--iters', type=int, default=50)
    ap.add_argument('--steps', type=int, default=5)
    ap.add_argument('--rounds', type=int, default=3)
    ap.add_argument('--no-step', action='store_true')
    args = ap.parse_args()
    assert torch.cuda.is_available(), 'the timing needs a GPU'
    meta = card()
    for P in args.pairs:
        bench_kernel(P, args.iters, args.rounds + 2, meta)
    if not args.no_step:
        bench_step(args.steps, args.rounds, meta)


if __name__ == '__main__':
    main()
