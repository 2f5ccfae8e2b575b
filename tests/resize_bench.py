"""Time the colour-frame resize of one scan, 20 views 640x480 -> 480x480 (ScanNet frames at the configs' Resize scale),
on the GPU (esb_img_resize_linear_u8, one launch for all views) and with cv2.resize on one host thread per frame.

GPU: each timed window is `--launches` back-to-back calls into a preallocated output between two CUDA events, after a
warm-up window; the median window over `--rounds` gives the time per call. Achieved bandwidth counts the algorithmic
bytes, V*H*W*3 read plus V*h*w*3 written. cv2 (when installed): the 20 frames resized one after another with
cv2.setNumThreads(1), median over the rounds. The card's name and power limit are read in the same process. Prints one
JSON object; DESIGN §6 quotes it.

  python tests/resize_bench.py [--rounds 7] [--launches 200]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from embodiedscan_b200._ffi import call, ptr, stream  # noqa: E402
from embodiedscan_b200.transforms import resize_multiview  # noqa: E402

V, H, W, h, w = 20, 480, 640, 480, 480
HBM_BYTES_PER_S = 3.35e12          # H100 SXM data sheet


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--rounds', type=int, default=7)
    ap.add_argument('--launches', type=int, default=200)
    args = ap.parse_args()
    assert torch.cuda.is_available(), 'resize_bench.py times the kernel on a GPU'
    frames = np.random.RandomState(0).randint(0, 256, size=(V, H, W, 3), dtype=np.uint8)
    src = torch.from_numpy(frames).cuda()
    out = torch.empty((V, 3, h, w), dtype=torch.uint8, device=src.device)

    def window(n):
        t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        t0.record()
        for _ in range(n):
            call('esb_img_resize_linear_u8', ptr(src), V, H, W, h, w, ptr(out), stream())
        t1.record()
        t1.synchronize()
        return t0.elapsed_time(t1) * 1e-3 / n

    window(args.launches)
    gpu = sorted(window(args.launches) for _ in range(args.rounds))
    med = gpu[len(gpu) // 2]
    # one call as a caller makes it (output allocated per call), host clock around a synchronised call
    for _ in range(10):
        resize_multiview(src, (w, h))
    torch.cuda.synchronize()
    single = []
    for _ in range(args.rounds * 10):
        t = time.perf_counter()
        resize_multiview(src, (w, h))
        torch.cuda.synchronize()
        single.append(time.perf_counter() - t)
    single.sort()
    nbytes = V * H * W * 3 + V * h * w * 3
    res = {
        'workload': f'{V} views {W}x{H} -> {w}x{h}, uint8 HWC -> CHW',
        'bytes': nbytes,
        'gpu_us_per_call': round(med * 1e6, 2),
        'gpu_us_per_call_rounds': [round(t * 1e6, 2) for t in gpu],
        'gpu_achieved_TB_per_s': round(nbytes / med / 1e12, 3),
        'gpu_share_of_datasheet_hbm': round(nbytes / HBM_BYTES_PER_S / med, 3),
        'gpu_us_per_synchronised_call': round(single[len(single) // 2] * 1e6, 2),
    }
    try:
        import cv2
    except ImportError:
        res['cv2'] = 'not installed'
    else:
        cv2.setNumThreads(1)
        host = []
        for r in range(args.rounds + 1):
            t = time.perf_counter()
            for f in frames:
                cv2.resize(f, (w, h), interpolation=cv2.INTER_LINEAR)
            if r:                                          # round 0 warms up
                host.append(time.perf_counter() - t)
        host.sort()
        res['cv2'] = cv2.__version__
        res['cv2_one_thread_ms_per_scan'] = round(host[len(host) // 2] * 1e3, 3)
        res['cv2_one_thread_ms_per_scan_rounds'] = [round(t * 1e3, 3) for t in host]
        res['speedup_vs_cv2_one_thread'] = round(host[len(host) // 2] / med, 1)
    smi = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'],
                         capture_output=True, text=True).stdout.strip().splitlines()
    res['gpu'] = smi[0] if smi else torch.cuda.get_device_name()
    print(json.dumps(res, indent=1))


if __name__ == '__main__':
    main()
