"""Runs every case of test_sparse_bf16_gpu.py in this fresh interpreter with the profiler on and prints one JSON line,
{case label: the sparse-branch kernel instances the case launched}; the test module reads it to check each case's claim.
A case whose own checks fail still reports what it launched (the parent run reports the failure)."""
import json
import os
import sys
import traceback

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import test_sparse_bf16_gpu as T  # noqa: E402


def _calls(fn):
    """Keyword sets of a test function's parametrize marks (their cartesian product)."""
    combos = [{}]
    for m in getattr(fn, 'pytestmark', []):
        if m.name != 'parametrize':
            continue
        names = [n.strip() for n in m.args[0].split(',')]
        combos = [dict(c, **dict(zip(names, v if len(names) > 1 else (v, )))) for c in combos for v in m.args[1]]
    return combos


def main():
    T._CHILD = {}
    tests = [n for n in dir(T) if n.startswith('test_') and n != 'test_c2_step_launches_only_pinned_instances']
    for name in tests + ['test_c2_step_launches_only_pinned_instances']:
        for kw in _calls(getattr(T, name)):
            try:
                getattr(T, name)(**kw)
            except Exception:
                traceback.print_exc(file=sys.stderr)
    print(json.dumps(T._CHILD))


if __name__ == '__main__':
    main()
