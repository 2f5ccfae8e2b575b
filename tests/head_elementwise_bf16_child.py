"""Runs every case of test_head_elementwise_bf16_gpu.py in this fresh interpreter with the profiler on and prints one JSON
line, {case label: the library kernel instances the case launched}; the test module reads it to check each case's claim.
A case whose own checks fail still reports what it launched (the parent run reports the failure)."""
import json
import os
import sys
import traceback

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import test_head_elementwise_bf16_gpu as T  # noqa: E402
from sparse_bf16_child import _calls  # noqa: E402


def main():
    T._CHILD = {}
    census = 'test_step_launches_only_held_library_kernels'
    tests = [n for n in dir(T) if n.startswith('test_') and n != census and not getattr(getattr(T, n), 'no_child', False)]
    for name in tests + [census]:
        for kw in _calls(getattr(T, name)):
            try:
                getattr(T, name)(**kw)
            except Exception:
                traceback.print_exc(file=sys.stderr)
    print(json.dumps(T._CHILD))


if __name__ == '__main__':
    main()
