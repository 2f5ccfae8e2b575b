"""Runs every case of test_dense_bf16_gpu.py in this fresh interpreter with the profiler on and prints one JSON line,
{case label: the dense-branch kernel instances the case launched}; the test module reads it to check each case's claim.
A case whose own checks fail still reports what it launched (the parent run reports the failure)."""
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import test_dense_bf16_gpu as T  # noqa: E402
from sparse_bf16_child import run_cases  # noqa: E402


def main():
    census = 'test_step_launches_only_pinned_dense_instances'
    tests = [n for n in dir(T) if n.startswith('test_') and n != census]
    print(json.dumps(run_cases(T, tests + [census])))


if __name__ == '__main__':
    main()
