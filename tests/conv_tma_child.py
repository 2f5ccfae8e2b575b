"""C2-sized timings of the TMA + wgmma conv2d kernels (csrc/conv_tma.cu) against cuDNN, and of the 7x7 stem: one JSON line
per layer. Run with `--bench`; correctness is pinned per element by tests/test_dense_bf16_gpu.py."""
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import torch  # noqa: E402
import torch.nn.functional as F  # noqa: E402


def bench_stem(dev):
    from embodiedscan_b200.backbones import _ConvBlock2D
    x = torch.randn(80, 3, 480, 640, device=dev).bfloat16().contiguous(memory_format=torch.channels_last)
    w = torch.randn(16, 3, 7, 7, device=dev).bfloat16().contiguous(memory_format=torch.channels_last)
    b = torch.zeros(16, device=dev)
    for _ in range(3):
        _ConvBlock2D.apply(x, w, b, None, True, 2, 3)
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(10):
        y = _ConvBlock2D.apply(x, w, b, None, True, 2, 3)
    e1.record()
    torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / 10
    print(json.dumps(dict(kind='bench_stem', us=1e3 * ms, gbs=(x.numel() + y.numel()) * 2 / ms / 1e6)), flush=True)


# the convolutions of ResNet-50/16 at C2 (80 views of 480x640 per step): cin, cout, k, stride, pad, (H, W) of the input
BENCH = [
    (16, 16, 1, 1, 0, (120, 160)), (16, 16, 3, 1, 1, (120, 160)), (16, 64, 1, 1, 0, (120, 160)), (64, 16, 1, 1, 0, (120, 160)),
    (64, 32, 1, 1, 0, (120, 160)), (32, 32, 3, 2, 1, (120, 160)), (32, 128, 1, 1, 0, (60, 80)), (128, 32, 1, 1, 0, (60, 80)),
    (32, 32, 3, 1, 1, (60, 80)), (64, 64, 3, 1, 1, (30, 40)), (64, 256, 1, 1, 0, (30, 40)), (256, 64, 1, 1, 0, (30, 40)),
    (128, 128, 3, 1, 1, (15, 20)), (128, 512, 1, 1, 0, (15, 20)), (512, 128, 1, 1, 0, (15, 20)),
]


def bench(dev, n=80):
    from embodiedscan_b200.backbones import conv2d_tma, ohwi
    for cin, cout, k, stride, pad, hw in BENCH:
        x = torch.randn(n, cin, *hw, device=dev).bfloat16().contiguous(memory_format=torch.channels_last)
        w = torch.randn(cout, cin, k, k, device=dev).bfloat16()
        wd = ohwi(w)
        b = torch.zeros(cout, device=dev)
        wcl = w.contiguous(memory_format=torch.channels_last)
        ms = {}
        for name, fn in (('tma', lambda: conv2d_tma(x, wd, b, None, True, stride, pad)),
                         ('cudnn', lambda: F.relu(F.conv2d(x, wcl, None, stride, pad)))):
            for _ in range(3):
                y = fn()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(10):
                y = fn()
            e1.record()
            torch.cuda.synchronize()
            ms[name] = e0.elapsed_time(e1) / 10
        byt = (x.numel() + y.numel() + w.numel()) * 2
        from embodiedscan_b200.backbones import conv2d_tma_wgrad
        dyb = torch.randn_like(y)
        for _ in range(2):
            conv2d_tma_wgrad(x, dyb, tuple(w.shape), stride, pad)
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(5):
            conv2d_tma_wgrad(x, dyb, tuple(w.shape), stride, pad)
        e1.record()
        torch.cuda.synchronize()
        ms['wgrad_tma'] = e0.elapsed_time(e1) / 5
        print(json.dumps(dict(kind='bench', case=[cin, cout, k, stride, pad, list(hw), n], us_tma=1e3 * ms['tma'],
                              us_cudnn=1e3 * ms['cudnn'], gbs_tma=byt / ms['tma'] / 1e6, mbytes=byt / 1e6,
                              us_wgrad_tma=1e3 * ms['wgrad_tma'], gbs_wgrad_tma=byt / ms['wgrad_tma'] / 1e6)), flush=True)


def main():
    if '--bench' in sys.argv:
        dev = 'cuda:0'
        bench_stem(dev)
        bench(dev)


if __name__ == '__main__':
    main()
