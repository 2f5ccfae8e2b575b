"""Time the AdamW launch (esb_adamw_step_groups, without the clip-norm launch) over an arena of the C2 detector's size,
with 1, 8, one-per-parameter and 2048 parameter groups: median of 5 CUDA-event windows of 100 back-to-back launches.
Prints one JSON object; DESIGN §6 quotes it.

  python tests/optim_bench.py
"""
import json
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from embodiedscan_b200 import MODELS, _ffi  # noqa: E402
from embodiedscan_b200.engine import ALIGN  # noqa: E402
from embodiedscan_b200.synth import mv_det3d_config  # noqa: E402


def main():
    assert torch.cuda.is_available(), 'optim_bench.py times the kernel on a GPU'
    model = MODELS.build(mv_det3d_config('C2'))
    sizes = [(p.numel() + ALIGN - 1) // ALIGN * ALIGN for p in model.parameters() if p.requires_grad]
    del model
    n = sum(sizes)
    offs = np.cumsum([0] + sizes)
    torch.manual_seed(0)
    p, g, m = (torch.randn(n, device='cuda') * 1e-2 for _ in range(3))
    v = torch.rand(n, device='cuda') * 1e-4
    clip = torch.tensor([0., 0., 1.], device='cuda')
    out = {'gpu': torch.cuda.get_device_name(), 'n_params': len(sizes), 'n_elements': n}
    for label, G in (('1 group', 1), ('8 groups', 8), (f'{len(sizes)} groups (one per parameter)', len(sizes)),
                     ('2048 groups (equal slices)', 2048)):
        idx = None
        if G > 1:
            a = np.zeros(n, dtype=np.uint16)
            if G <= len(sizes):
                for k in range(len(sizes)):
                    a[offs[k]:offs[k + 1]] = k % G
            else:
                a[:] = (np.arange(n) * G // n).astype(np.uint16)
            idx = torch.from_numpy(a).cuda()
        lr_wd = torch.tensor([x for k in range(G) for x in (1e-3 * (1 + k % 3), 1e-4)], dtype=torch.float32)

        def launch():
            _ffi.call('esb_adamw_step_groups', p.data_ptr(), g.data_ptr(), m.data_ptr(), v.data_ptr(), _ffi.ptr(idx),
                      lr_wd.data_ptr(), G, n, 0.9, 0.999, 1e-8, 1, 1.0, clip.data_ptr(), _ffi.stream())
        for _ in range(20):
            launch()
        reps = []
        for _ in range(5):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(100):
                launch()
            e1.record()
            torch.cuda.synchronize()
            reps.append(e0.elapsed_time(e1) / 100)
        ms = sorted(reps)[len(reps) // 2]
        by = n * (28 + (2 if G > 1 else 0))
        out[label] = {'ms': ms, 'ms_windows': reps, 'bytes': by, 'TB_s': by / ms / 1e9}
    print(json.dumps(out, indent=1))


if __name__ == '__main__':
    main()
