"""Timing of the chamfer_distance kernels (csrc/chamfer.cu); pytest does not collect this file.

    python tests/chamfer_child.py --bench [--n 16384] [--b 4] [--iters 20]

Prints one JSON line per criterion at B x N x N points with C = 3: forward (both directions) and backward kernel times
from CUDA events after warm-up, pair evaluations per second, the chunked-ATen restatement of the reference timed in
the same run, and the card name and power limit."""
import argparse
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))


def _time_ms(fn, iters):
    start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    times = []
    for _ in range(iters):
        start.record()
        fn()
        end.record()
        torch.cuda.synchronize()
        times.append(start.elapsed_time(end))
    times.sort()
    return times[len(times) // 2]


def _power_limit_w():
    try:
        out = subprocess.run(['nvidia-smi', '--query-gpu=power.limit', '--format=csv,noheader,nounits', '-i',
                              str(torch.cuda.current_device())], capture_output=True, text=True, timeout=30)
        return float(out.stdout.strip().splitlines()[0])
    except Exception:
        return None


def bench(B, N, iters):
    from embodiedscan_b200 import _ffi
    from embodiedscan_b200.dense_heads import _CD_MODE_CODE
    from losses_util import nearest
    g = torch.Generator(device='cuda').manual_seed(0)
    src = torch.rand(B, N, 3, device='cuda', generator=g) * 4 - 2
    dst = torch.rand(B, N, 3, device='cuda', generator=g) * 4 - 2
    d1, d2 = torch.empty(B, N, device='cuda'), torch.empty(B, N, device='cuda')
    i1, i2 = torch.empty(B, N, dtype=torch.int64, device='cuda'), torch.empty(B, N, dtype=torch.int64, device='cuda')
    g1, g2 = torch.rand(B, N, device='cuda'), torch.rand(B, N, device='cuda')
    gs, gd = torch.empty_like(src), torch.empty_like(dst)
    card = torch.cuda.get_device_name()
    power = _power_limit_w()
    for mode in ('l1', 'l2', 'smooth_l1'):
        m = _CD_MODE_CODE[mode]

        def fwd():
            _ffi.call('esb_chamfer_fwd', src.data_ptr(), dst.data_ptr(), B, N, N, 3, m, d1.data_ptr(), d2.data_ptr(),
                      i1.data_ptr(), i2.data_ptr(), _ffi.stream())

        def bwd():
            _ffi.call('esb_chamfer_bwd', src.data_ptr(), dst.data_ptr(), i1.data_ptr(), i2.data_ptr(), g1.data_ptr(),
                      g2.data_ptr(), B, N, N, 3, m, gs.data_ptr(), gd.data_ptr(), _ffi.stream())

        def ref():
            nearest(src, dst, mode, chunk=1024)
            nearest(dst, src, mode, chunk=1024)

        for f in (fwd, bwd, ref):
            f()
        torch.cuda.synchronize()
        fwd_ms, bwd_ms = _time_ms(fwd, iters), _time_ms(bwd, iters)
        ref_ms = _time_ms(ref, max(3, iters // 5))
        pairs = 2.0 * B * N * N
        print(json.dumps(dict(mode=mode, B=B, N=N, M=N, C=3, fwd_ms=round(fwd_ms, 4), bwd_ms=round(bwd_ms, 4),
                              pairs_per_s=pairs / (fwd_ms * 1e-3), aten_chunked_fwd_ms=round(ref_ms, 3),
                              speedup_vs_aten=round(ref_ms / fwd_ms, 1), card=card, power_limit_w=power)), flush=True)


if __name__ == '__main__':
    ap = argparse.ArgumentParser()
    ap.add_argument('--bench', action='store_true')
    ap.add_argument('--b', type=int, default=4)
    ap.add_argument('--n', type=int, default=16384)
    ap.add_argument('--iters', type=int, default=20)
    a = ap.parse_args()
    if a.bench:
        bench(a.b, a.n, a.iters)
