"""Child process: the wgmma flash-attention kernels (csrc/attn_tc.cu) against fp32 softmax attention on the bf16-rounded
operands, forward and backward, with and without a key padding mask; one JSON line per case, `--bench` adds timings."""
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import torch  # noqa: E402


def ref_attn(q, k, v, pad, scale):
    s = (q @ k.transpose(-1, -2)) * scale
    if pad is not None:
        s = s.masked_fill(pad[:, None, None, :], float('-inf'))
    p = torch.softmax(s, -1)
    p = torch.nan_to_num(p, nan=0.0)                  # a query whose keys are all padded: zero output
    return p @ v


def run(B, H, Lq, Lk, masked, dev):
    from embodiedscan_b200.grounding import flash_attention
    g = torch.Generator().manual_seed(B * 1000 + Lq + Lk)
    q, k, v = (torch.randn(B, H, L, 32, generator=g).bfloat16() for L in (Lq, Lk, Lk))
    pad = None
    if masked:
        lens = torch.randint(max(Lk // 3, 1), Lk + 1, (B, ), generator=g)
        pad = torch.arange(Lk)[None, :] >= lens[:, None]
    scale = 32 ** -0.5
    qr, kr, vr = (t.float().requires_grad_(True) for t in (q, k, v))
    ref = ref_attn(qr, kr, vr, pad, scale)
    go = torch.randn(ref.shape, generator=g).bfloat16()
    ref.backward(go.float())
    qd, kd, vd = (t.to(dev).requires_grad_(True) for t in (q, k, v))
    out = flash_attention(qd, kd, vd, pad.to(dev) if pad is not None else None, scale)
    out.backward(go.to(dev))
    torch.cuda.synchronize()
    res = dict(kind='attn', case=[B, H, Lq, Lk, masked])
    ok = True
    for name, a, b_ in (('fwd', out, ref), ('dq', qd.grad, qr.grad), ('dk', kd.grad, kr.grad), ('dv', vd.grad, vr.grad)):
        err = float((a.float().cpu() - b_.detach()).abs().max())
        tol = 2e-2 * max(float(b_.detach().abs().max()), 1e-3)
        res[name] = err
        ok = ok and err <= tol and bool(torch.isfinite(a).all())
    res['ok'] = ok
    print(json.dumps(res), flush=True)


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


if __name__ == '__main__':
    dev = 'cuda:0'
    for case in ((1, 1, 128, 128, False), (2, 8, 256, 256, False), (2, 8, 256, 300, True), (3, 8, 256, 1000, True),
                 (1, 8, 200, 3500, True), (2, 2, 77, 19, True)):
        try:
            run(*case, dev)
        except Exception as e:  # noqa
            print(json.dumps(dict(kind='error', case=list(case), ok=False, err=str(e)[:300])), flush=True)
    if '--bench' in sys.argv:
        bench(dev)
