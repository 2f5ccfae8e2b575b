"""Child process of tests/test_a_golden_gpu.py::test_conv2d_tc_forward_matches_torch: runs the experimental wgmma conv2d
kernel against torch's fp32 convolution on bf16-rounded inputs and prints one JSON line per case."""
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import torch  # noqa: E402
import torch.nn.functional as F  # noqa: E402

CASES = [
    (16, 16, 1, 1, 0, (30, 40), 3, False),      # thin 1x1: one 64-wide chunk, 16 valid reduction elements, N_TILE 32
    (16, 16, 3, 1, 1, (30, 40), 3, False),      # 3x3x16: 4 taps per chunk, 3 chunks (the last one 1/4 full)
    (16, 64, 1, 1, 0, (30, 40), 3, True),       # bottleneck expansion + residual + ReLU
    (64, 128, 1, 2, 0, (30, 40), 2, False),     # strided 1x1 (downsample branch)
    (32, 32, 3, 2, 1, (31, 41), 2, False),      # strided 3x3 on odd sizes (pixel rows not a multiple of 128)
    (128, 512, 1, 1, 0, (15, 20), 8, True),     # N_TILE 256 / two channel tiles
    (8, 16, 7, 2, 3, (48, 64), 2, False),       # stem geometry on an 8-channel padded input
]


def main():
    from embodiedscan_b200.backbones import conv2d_tc, conv2d_tc_dgrad, conv2d_tc_wgrad, pack_ohwi
    dev = 'cuda:0'
    for cin, cout, k, stride, pad, hw, n, with_res in CASES:
        g = torch.Generator().manual_seed(cin * 1000 + cout + k)
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
        out = conv2d_tc(xd, pack_ohwi(w.to(dev)), b.to(dev), rd, True, k, k, stride, pad)
        torch.cuda.synchronize()
        err = float((out.float().cpu() - ref).abs().max())
        tol = 2e-2 * max(float(ref.abs().max()), 1.0)
        print(json.dumps(dict(kind='fwd', case=[cin, cout, k, stride, pad, list(hw), n, with_res], err=err, tol=tol,
                              ok=bool(out.shape == ref.shape and err <= tol))), flush=True)
        if cin == 8:
            continue                                     # the stem is frozen: no input gradient on the path
        # input gradient through the transposed-gather mode of the same kernel
        xr = x.float().requires_grad_(True)
        yr = F.conv2d(xr, w.float(), None, stride, pad)
        dy = torch.randn(yr.shape, generator=g).bfloat16()
        yr.backward(dy.float())
        dx = conv2d_tc_dgrad(dy.to(dev).contiguous(memory_format=torch.channels_last), w.to(dev), hw, stride, pad)
        torch.cuda.synchronize()
        err = float((dx.float().cpu() - xr.grad).abs().max())
        tol = 2e-2 * max(float(xr.grad.abs().max()), 1.0)
        print(json.dumps(dict(kind='dgrad', case=[cin, cout, k, stride, pad, list(hw), n], err=err, tol=tol,
                              ok=bool(dx.shape == xr.grad.shape and err <= tol))), flush=True)
        # weight gradient (pixels are the reduction dimension)
        wr = w.float().requires_grad_(True)
        F.conv2d(x.float(), wr, None, stride, pad).backward(dy.float())
        dw = conv2d_tc_wgrad(xd, dy.to(dev).contiguous(memory_format=torch.channels_last), tuple(w.shape), stride, pad)
        torch.cuda.synchronize()
        err = float((dw.float().cpu() - wr.grad).abs().max())
        tol = 2e-2 * max(float(wr.grad.abs().max()), 1.0)
        print(json.dumps(dict(kind='wgrad', case=[cin, cout, k, stride, pad, list(hw), n], err=err, tol=tol,
                              ok=bool(tuple(dw.shape) == tuple(wr.grad.shape) and err <= tol))), flush=True)


if __name__ == '__main__':
    main()
