"""Child process of tests/test_kernels_gpu.py::test_conv2d_tma_*: runs the TMA + wgmma conv2d kernel (csrc/conv_tma.cu)
against torch's fp32 convolution on bf16-rounded inputs, one JSON line per case (a first-run tensor-core kernel that hangs
must not take the test session with it: the parent applies a timeout).  `--bench` adds C2-sized timings."""
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import torch  # noqa: E402
import torch.nn.functional as F  # noqa: E402

# cin, cout, k, stride, pad, (H, W), n_img, residual
CASES = [
    (64, 16, 1, 1, 0, (30, 40), 3, False),      # 1x1 squeeze: one 128B-swizzled chunk, N = 16
    (16, 16, 3, 1, 1, (30, 40), 3, False),      # 3x3x16: 32B swizzle, 4 taps per stage, 9 taps = 3 stages (last 1/4 full)
    (16, 64, 1, 1, 0, (30, 40), 3, True),       # bottleneck expansion + residual + ReLU
    (32, 32, 3, 1, 1, (17, 23), 2, False),      # 64B swizzle, 2 taps per stage, odd extent (clipped stores)
    (64, 64, 3, 1, 1, (30, 40), 2, False),      # 128B swizzle, one tap per stage
    (128, 128, 3, 1, 1, (15, 20), 5, False),    # two channel chunks per tap; whole images per tile (TN > 1)
    (64, 128, 1, 2, 0, (30, 40), 2, False),     # strided 1x1 (downsample branch): tensor-map element strides
    (32, 32, 3, 2, 1, (31, 41), 2, False),      # strided 3x3 on odd sizes
    (256, 512, 1, 1, 0, (15, 20), 4, True),     # N_TILE 256, two channel blocks
    (512, 128, 1, 1, 0, (15, 20), 4, False),    # 8 chunks of reduction
    (16, 16, 1, 1, 0, (120, 160), 2, False),    # many tiles per CTA (persistent loop, both accumulator stages)
]


def run_stem(dev):
    """The 7x7/2 stem (wgmma with shared-memory im2col) through the module-level dispatch of backbones._ConvBlock2D."""
    from embodiedscan_b200.backbones import _ConvBlock2D
    for n, hw in ((2, (48, 64)), (3, (62, 90)), (1, (480, 640))):
        g = torch.Generator().manual_seed(n * 7 + hw[0])
        x = torch.randn(n, 3, *hw, generator=g).bfloat16()
        w = (torch.randn(16, 3, 7, 7, generator=g) / 147 ** 0.5).bfloat16()
        b = torch.randn(16, generator=g)
        ref = F.relu(F.conv2d(x.float(), w.float(), b, 2, 3))
        out = _ConvBlock2D.apply(x.to(dev).contiguous(memory_format=torch.channels_last),
                                 w.to(dev).contiguous(memory_format=torch.channels_last), b.to(dev), None, True, 2, 3)
        torch.cuda.synchronize()
        err = float((out.float().cpu() - ref).abs().max())
        tol = 1e-2 * max(float(ref.abs().max()), 1.0)
        print(json.dumps(dict(kind='stem', case=[n, list(hw)], err=err, tol=tol, ok=bool(out.shape == ref.shape and err <= tol))),
              flush=True)
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


def run_conv3d(dev):
    """Rank-5 tensor maps: nn.Conv3d forward / dgrad (stride 1, 2) / wgrad and the k2 s2 transpose of the occupancy neck
    through occupancy._conv3d, against torch fp32 on bf16-rounded operands."""
    import torch.nn as nn
    from embodiedscan_b200.occupancy import _conv3d
    cases = [(64, 64, 3, 1, 1, (6, 10, 8), 2), (64, 128, 3, 2, 1, (6, 10, 8), 2), (128, 256, 1, 2, 0, (6, 10, 8), 1),
             (256, 256, 3, 1, 1, (4, 5, 5), 1), (768, 256, 3, 1, 1, (4, 6, 5), 1), (128, 64, 2, 2, 0, (3, 5, 4), 2)]
    for cin, cout, k, stride, pad, dhw, n in cases:
        g = torch.Generator().manual_seed(cin + cout + k)
        transpose = k == 2
        conv = (nn.ConvTranspose3d(cin, cout, 2, 2, bias=False) if transpose else nn.Conv3d(cin, cout, k, stride, pad, bias=False))
        with torch.no_grad():
            conv.weight.copy_((torch.randn(conv.weight.shape, generator=g) / (cin * k ** 3) ** 0.5).bfloat16().float())
        x = torch.randn(n, cin, *dhw, generator=g).bfloat16()
        xr = x.float().requires_grad_(True)
        ref = conv(xr)
        go = torch.randn(ref.shape, generator=g).bfloat16()
        ref.backward(go.float())
        wref = conv.weight.grad.clone()
        conv.weight.grad = None
        convd = conv.to(dev)
        xd = x.to(dev).contiguous(memory_format=torch.channels_last_3d).requires_grad_(True)
        out = _conv3d(convd, xd)
        out.backward(go.to(dev))
        torch.cuda.synchronize()
        res = dict(kind='conv3d', case=[cin, cout, k, stride, pad, list(dhw), n])
        ok = tuple(out.shape) == tuple(ref.shape)
        for name, a, b in (('fwd', out, ref), ('dgrad', xd.grad, xr.grad), ('wgrad', convd.weight.grad, wref)):
            err = float((a.float().cpu() - b.detach()).abs().max())
            tol = 1e-2 * max(float(b.detach().abs().max()), 1.0)
            res[name] = err
            ok = ok and err <= tol
        res['ok'] = bool(ok)
        print(json.dumps(res), flush=True)


def run_dispatch(dev):
    """A bf16 convolution with TMA-sized channels and stride 3 through backbones._ConvBlock2D, forward and backward: the
    TMA forward and wgrad, and the dgrad of csrc/conv2d_direct.cu (the TMA dgrad takes strides 1 and 2 only), against
    torch fp32 on bf16-rounded operands."""
    from embodiedscan_b200.backbones import _ConvBlock2D
    cin, cout, k, stride, pad, hw, n = 64, 64, 3, 3, 1, (31, 41), 2
    g = torch.Generator().manual_seed(3)
    x = torch.randn(n, cin, *hw, generator=g).bfloat16()
    w = (torch.randn(cout, cin, k, k, generator=g) / (cin * k * k) ** 0.5).bfloat16()
    b = torch.randn(cout, generator=g)
    xr, wr = x.float().requires_grad_(True), w.float().requires_grad_(True)
    ref = F.conv2d(xr, wr, b, stride, pad)
    dy = torch.randn(ref.shape, generator=g).bfloat16()
    ref.backward(dy.float())
    xd = x.to(dev).contiguous(memory_format=torch.channels_last).requires_grad_(True)
    wd = w.to(dev).contiguous(memory_format=torch.channels_last).requires_grad_(True)
    out = _ConvBlock2D.apply(xd, wd, b.to(dev), None, False, stride, pad)
    out.backward(dy.to(dev).contiguous(memory_format=torch.channels_last))
    torch.cuda.synchronize()
    res = dict(kind='dispatch', case=[cin, cout, k, stride, pad, list(hw), n])
    ok = tuple(out.shape) == tuple(ref.shape)
    for name, a, r in (('fwd', out, ref), ('dgrad', xd.grad, xr.grad), ('wgrad', wd.grad, wr.grad)):
        err = float((a.float().cpu() - r.detach()).abs().max())
        tol = 1e-2 * max(float(r.detach().abs().max()), 1.0)
        res[name] = err
        ok = ok and err <= tol
    res['ok'] = bool(ok)
    print(json.dumps(res), flush=True)


def run_case(case, dev):
    from embodiedscan_b200.backbones import conv2d_tma, conv2d_tma_dgrad, ohwi
    cin, cout, k, stride, pad, hw, n, with_res = case
    g = torch.Generator().manual_seed(cin * 1000 + cout + k + stride)
    x = torch.randn(n, cin, *hw, generator=g).bfloat16()
    w = (torch.randn(cout, cin, k, k, generator=g) / (cin * k * k) ** 0.5).bfloat16()
    b = torch.randn(cout, generator=g)
    ref = F.conv2d(x.float(), w.float(), b, stride, pad)
    res = torch.randn(ref.shape, generator=g).bfloat16() if with_res else None
    if with_res:
        ref = ref + res.float()
    ref = F.relu(ref)
    xd = x.to(dev).contiguous(memory_format=torch.channels_last)
    rd = res.to(dev).contiguous(memory_format=torch.channels_last) if with_res else None
    wd = ohwi(w.to(dev))
    out = conv2d_tma(xd, wd, b.to(dev), rd, True, stride, pad)
    torch.cuda.synchronize()
    err = float((out.float().cpu() - ref).abs().max())
    tol = 1e-2 * max(float(ref.abs().max()), 1.0)            # bf16 output rounding of values up to |max|
    print(json.dumps(dict(kind='fwd', case=list(case[:5]) + [list(hw), n, with_res], err=err, tol=tol,
                          ok=bool(out.shape == ref.shape and err <= tol))), flush=True)
    # weight gradient (TMA-fed, pixels are the reduction dimension)
    from embodiedscan_b200.backbones import conv2d_tma_wgrad
    wr = w.float().requires_grad_(True)
    yw = F.conv2d(x.float(), wr, None, stride, pad)
    dyw = torch.randn(yw.shape, generator=g).bfloat16()
    yw.backward(dyw.float())
    dw = conv2d_tma_wgrad(xd, dyw.to(dev).contiguous(memory_format=torch.channels_last), tuple(w.shape), stride, pad)
    torch.cuda.synchronize()
    err = float((dw.float().cpu() - wr.grad).abs().max())
    tol = 1e-2 * max(float(wr.grad.abs().max()), 1.0)
    print(json.dumps(dict(kind='wgrad', case=list(case[:5]) + [list(hw), n], err=err, tol=tol,
                          ok=bool(tuple(dw.shape) == tuple(wr.grad.shape) and err <= tol))), flush=True)
    if stride not in (1, 2):
        return
    xr = x.float().requires_grad_(True)
    yr = F.conv2d(xr, w.float(), None, stride, pad)
    dy = torch.randn(yr.shape, generator=g).bfloat16()
    yr.backward(dy.float())
    dx = conv2d_tma_dgrad(dy.to(dev).contiguous(memory_format=torch.channels_last), wd, hw, pad, stride)
    torch.cuda.synchronize()
    err = float((dx.float().cpu() - xr.grad).abs().max())
    tol = 1e-2 * max(float(xr.grad.abs().max()), 1.0)
    print(json.dumps(dict(kind='dgrad', case=list(case[:5]) + [list(hw), n], err=err, tol=tol,
                          ok=bool(dx.shape == xr.grad.shape and err <= tol))), flush=True)


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
    dev = 'cuda:0'
    only = [int(a) for a in sys.argv[1:] if a.isdigit()]
    for i, case in enumerate(CASES):
        if only and i not in only:
            continue
        try:
            run_case(case, dev)
        except Exception as e:  # noqa
            print(json.dumps(dict(kind='error', case=list(case[:5]), ok=False, err=str(e)[:300])), flush=True)
    try:
        run_stem(dev)
    except Exception as e:  # noqa
        print(json.dumps(dict(kind='error', case='stem', ok=False, err=str(e)[:300])), flush=True)
    if not only:
        try:
            run_dispatch(dev)
        except Exception as e:  # noqa
            print(json.dumps(dict(kind='error', case='dispatch', ok=False, err=str(e)[:300])), flush=True)
        try:
            run_conv3d(dev)
        except Exception as e:  # noqa
            import traceback
            print(json.dumps(dict(kind='error', case='conv3d', ok=False, err=traceback.format_exc()[-400:])), flush=True)
    if '--bench' in sys.argv:
        bench(dev)


if __name__ == '__main__':
    main()
