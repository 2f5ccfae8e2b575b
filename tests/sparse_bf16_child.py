"""Runs every case of test_sparse_bf16_gpu.py in this fresh interpreter with the profiler on and prints one JSON line,
{case label: the sparse-branch kernel instances the case launched}; the test module reads it to check each case's claim.
A case whose own checks fail still reports what it launched (the parent run reports the failure). Every case runs twice
(run_cases, shared with the dense and head / elementwise children)."""
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


def run_cases(T, names, passes=2):
    """Run the cases of the test functions `names` of module T (in that order, every parameter set) `passes` times, with
    T._CHILD set so that each case records what it launched, and return {case label: the union over the passes}. A short
    profiler session now and then records no event for a kernel it ran (the only kernel of the session, or one of a few),
    and the case's claim then fails although the kernel ran. Each case builds its operands anew, so running it again is
    safe, and a claimed instance is reported missing only when every pass missed it."""
    launched = {}
    for _ in range(passes):
        T._CHILD = {}
        for name in names:
            for kw in _calls(getattr(T, name)):
                try:
                    getattr(T, name)(**kw)
                except Exception:
                    traceback.print_exc(file=sys.stderr)
        for what, seen in T._CHILD.items():
            launched[what] = sorted(set(launched.get(what, ())) | set(seen))
    return launched


def main():
    census = 'test_c2_step_launches_only_pinned_instances'
    tests = [n for n in dir(T) if n.startswith('test_') and n != census]
    print(json.dumps(run_cases(T, tests + [census])))


if __name__ == '__main__':
    main()
