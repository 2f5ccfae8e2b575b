"""Compile embodiedscan_b200/csrc/*.cu into the in-tree C-ABI library ``libesb200.so`` for sm_90a (H100).

nvcc cross-compiles without a GPU; the .so is git-ignored but travels to the GPU box with the snapshot.
"""
import concurrent.futures as cf
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, 'csrc')
LIB = os.path.join(HERE, 'libesb200.so')
OBJ_DIR = os.path.join(HERE, 'csrc', '_obj')
NVCC = os.environ.get('NVCC', '/usr/local/cuda/bin/nvcc')
FLAGS = [
    '-gencode', 'arch=compute_90a,code=sm_90a', '-lineinfo', '-O3', '-std=c++17', '-Xcompiler', '-fPIC',
    '--expt-relaxed-constexpr', '-Xptxas', '-v'
]


def sources():
    return sorted(os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith('.cu'))


def _stale(target, deps):
    if not os.path.exists(target):
        return True
    t = os.path.getmtime(target)
    return any(os.path.getmtime(d) > t for d in deps)


def _compile(src):
    obj = os.path.join(OBJ_DIR, os.path.basename(src)[:-3] + '.o')
    headers = [os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith(('.cuh', '.h'))]
    if not _stale(obj, [src] + headers):
        return obj, ''
    cmd = [NVCC] + FLAGS + ['-c', src, '-o', obj]
    p = subprocess.run(cmd, capture_output=True, text=True)
    if p.returncode != 0:
        raise RuntimeError(f'nvcc failed for {src}:\n{p.stdout}\n{p.stderr}')
    return obj, p.stderr


def build_library(force=False, verbose=False):
    os.makedirs(OBJ_DIR, exist_ok=True)
    srcs = sources()
    if force:
        for f in os.listdir(OBJ_DIR):
            os.remove(os.path.join(OBJ_DIR, f))
    with cf.ThreadPoolExecutor(max_workers=min(8, len(srcs))) as ex:
        results = list(ex.map(_compile, srcs))
    objs = [r[0] for r in results]
    if verbose:
        for _, log in results:
            if log:
                sys.stderr.write(log)
    if force or _stale(LIB, objs):
        cmd = [NVCC, '-shared', '-o', LIB] + objs + ['-gencode', 'arch=compute_90a,code=sm_90a', '-lcudart']
        p = subprocess.run(cmd, capture_output=True, text=True)
        if p.returncode != 0:
            raise RuntimeError(f'link failed:\n{p.stdout}\n{p.stderr}')
    return LIB


if __name__ == '__main__':
    print(build_library(force='--force' in sys.argv, verbose=True))
