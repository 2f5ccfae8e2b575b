"""Timings of the wgmma flash-attention kernels (csrc/attn_tc.cu) against scaled_dot_product_attention at the grounding
decoder's size, forward and backward: one JSON line. Run with `--bench`; correctness is pinned per element by
tests/test_dense_bf16_gpu.py."""
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import torch  # noqa: E402


def bench(dev):
    from embodiedscan_b200.grounding import flash_attention
    B, H, Lq, Lk = 12, 8, 256, 3500
    q, k, v = (torch.randn(B, H, L, 32, device=dev).bfloat16().requires_grad_(True) for L in (Lq, Lk, Lk))
    pad = torch.zeros(B, Lk, dtype=torch.bool, device=dev)
    go = torch.randn(B, H, Lq, 32, device=dev).bfloat16()
    ms = {}
    for name, fn in (('own', lambda: flash_attention(q, k, v, pad)),
                     ('sdpa', lambda: torch.nn.functional.scaled_dot_product_attention(q, k, v, attn_mask=~pad[:, None, None, :]))):
        for _ in range(3):
            fn().backward(go)
        e0, e1, e2 = (torch.cuda.Event(enable_timing=True) for _ in range(3))
        e0.record()
        outs = [fn() for _ in range(5)]
        e1.record()
        for o in outs:
            o.backward(go)
        e2.record()
        torch.cuda.synchronize()
        ms[name] = (e0.elapsed_time(e1) / 5, e1.elapsed_time(e2) / 5)
    flops = 4.0 * B * H * Lq * Lk * 32
    print(json.dumps(dict(kind='bench', case=[B, H, Lq, Lk], fwd_us_own=1e3 * ms['own'][0], bwd_us_own=1e3 * ms['own'][1],
                          fwd_us_sdpa=1e3 * ms['sdpa'][0], bwd_us_sdpa=1e3 * ms['sdpa'][1],
                          fwd_tflops_own=flops / ms['own'][0] / 1e9)), flush=True)


if __name__ == '__main__' and '--bench' in sys.argv:
    bench('cuda:0')
