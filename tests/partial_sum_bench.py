"""Time the fixed-order partial-sum finisher (esb_sum_partial_rows) at the (n_parts, width) shapes one C2 bf16 training step
calls it with, against the one-thread-per-column loop it replaced, compiled from the source below into a temporary
directory. Both run in this process on the same operands, in alternating CUDA-event windows of 200 back-to-back launches (10 for the three largest loss sums)
after warm-up; the median window is reported. The partials stay in the 50 MB L2 between launches, as they do in the step,
where the producing kernel has just written them. Bytes = the partials read + out read (accumulate) + out written.
Prints one JSON object; DESIGN §6 quotes it.

  python tests/partial_sum_bench.py
"""
import ctypes
import json
import os
import subprocess
import sys
import tempfile

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from embodiedscan_b200 import _ffi  # noqa: E402
from embodiedscan_b200.build import NVCC  # noqa: E402

HBM_TB_S = 3.35           # H100 SXM data sheet
SYMBOL = '_Z20esb_sum_partial_rowsPKfixPfiP11CUstream_st'
# (n_parts, width, accumulate, calls): every host call of one C2 bf16 training step (4 scans x 20 views 480x640, 100k
# points). Width 1: the focal and box loss sums (accumulate) and the clip norm's sum of squares; widths 64..1024: the sparse
# norm statistics (S * C, 2 * C) and backward sums; 5184: a conv wgrad. The 2D branch's backward replays as a CUDA graph and
# its finisher calls (conv wgrad, attention dQ) are not in this list.
SHAPES = [
    (443750, 1, 1, 1), (84348, 1, 1, 1), (10544, 1, 1, 1), (1318, 1, 1, 1), (1056, 1, 0, 1), (27, 1, 1, 1),
    (145, 64, 1, 14),
    (2376, 128, 1, 4), (1563, 128, 1, 2), (297, 128, 1, 2), (264, 128, 0, 7), (48, 128, 1, 18), (38, 128, 1, 2),
    (5, 128, 1, 2),
    (297, 256, 1, 4), (264, 256, 0, 4), (207, 256, 0, 2), (207, 256, 1, 2), (191, 256, 0, 9), (149, 256, 0, 1),
    (19, 256, 0, 1), (15, 256, 1, 26),
    (264, 512, 0, 2), (59, 512, 0, 13), (38, 512, 1, 4), (5, 512, 1, 14),
    (149, 1024, 0, 2), (19, 1024, 0, 7),
    (19, 5184, 1, 1),
]

LOOP_SRC = r'''
#include <cuda_runtime.h>
__global__ void sum_partial_rows_loop(const float* __restrict__ part, int n_parts, long long width, float* __restrict__ out,
                                      int accumulate) {
  const long long j = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (j >= width) return;
  float s = accumulate ? out[j] : 0.f;
  for (int p = 0; p < n_parts; ++p) s += part[(long long)p * width + j];
  out[j] = s;
}
extern "C" int loop_sum_partial_rows(const float* part, int n_parts, long long width, float* out, int accumulate,
                                     cudaStream_t s) {
  sum_partial_rows_loop<<<(unsigned)((width + 255) / 256), 256, 0, s>>>(part, n_parts, width, out, accumulate);
  return (int)cudaPeekAtLastError();
}
'''


def _bind(fn):
    fn.argtypes = [ctypes.c_void_p, ctypes.c_int, ctypes.c_longlong, ctypes.c_void_p, ctypes.c_int, ctypes.c_void_p]
    fn.restype = ctypes.c_int
    return fn


def _loop_kernel(tmp):
    src, so = os.path.join(tmp, 'loop.cu'), os.path.join(tmp, 'libloop.so')
    with open(src, 'w') as f:
        f.write(LOOP_SRC)
    subprocess.run([NVCC, '-gencode', 'arch=compute_90a,code=sm_90a', '-O3', '-shared', '-Xcompiler', '-fPIC', src, '-o', so],
                   check=True)
    return _bind(ctypes.CDLL(so).loop_sum_partial_rows)


def _card():
    try:
        q = subprocess.run(['nvidia-smi', '-i', str(torch.cuda.current_device()), '--query-gpu=power.limit,clocks.max.sm',
                            '--format=csv,noheader'], capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        q = 'unknown'
    return {'gpu': torch.cuda.get_device_name(), 'power_limit, max SM clock': q}


def main():
    assert torch.cuda.is_available(), 'partial_sum_bench.py times the kernels on a GPU'
    new = _bind(getattr(_ffi.lib(), SYMBOL))
    with tempfile.TemporaryDirectory() as tmp:
        loop = _loop_kernel(tmp)
        out = _card()
        out['rows'] = []
        torch.manual_seed(0)
        st = _ffi.stream()
        for n_parts, width, acc, per_step in SHAPES:
            part = torch.randn(n_parts, width, device='cuda')
            res = {}
            for name, fn in (('loop', loop), ('tiled', new)):
                o = torch.randn(width, device='cuda')
                assert fn(part.data_ptr(), n_parts, width, o.data_ptr(), 0, st) == 0
                res[name] = o
            assert torch.equal(res['loop'].view(torch.int32), res['tiled'].view(torch.int32)), (n_parts, width)
            o = torch.zeros(width, device='cuda')
            windows = {'loop': [], 'tiled': []}
            reps = 200 if n_parts * width < 1 << 20 else 10
            for w in range(12):                          # alternate; the first two rounds are warm-up
                for name, fn in (('loop', loop), ('tiled', new)):
                    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                    e0.record()
                    for _ in range(reps):
                        fn(part.data_ptr(), n_parts, width, o.data_ptr(), acc, st)
                    e1.record()
                    torch.cuda.synchronize()
                    if w >= 2:
                        windows[name].append(e0.elapsed_time(e1) * 1e3 / reps)
            by = 4 * width * (n_parts + 1 + acc)
            row = {'n_parts': n_parts, 'width': width, 'accumulate': acc, 'calls_per_step': per_step,
                   'bytes': by}
            for name in ('loop', 'tiled'):
                us = sorted(windows[name])[len(windows[name]) // 2]
                row[name] = {'us': round(us, 2), 'TB_s': round(by / us / 1e6, 3), 'of_hbm': round(by / us / 1e6 / HBM_TB_S, 3)}
            row['speedup'] = round(row['loop']['us'] / row['tiled']['us'], 2)
            out['rows'].append(row)
        per_step = {name: sum(r[name]['us'] * r['calls_per_step'] for r in out['rows']) for name in ('loop', 'tiled')}
        out['us_per_step'] = {k: round(v, 1) for k, v in per_step.items()}
    print(json.dumps(out, indent=1))


if __name__ == '__main__':
    main()
