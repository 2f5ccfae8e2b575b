"""CPU: gradient accumulation on engine.OptimWrapper (`accumulative_counts`) — the micro-batch schedule against a
restatement of mmengine's OptimWrapper rules, and the data-parallel reducer over gloo (world 2): a non-syncing micro-batch
issues no collective, and after the window the arena holds the sum over ranks and micro-batches."""
import os
import sys
import warnings

import pytest
import torch
import torch.distributed as dist
import torch.nn as nn

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _mmengine_schedule(n, iters, init_counts=0, max_counts=None):
    """mmengine OptimWrapper (scale_loss / should_sync / backward / should_update), restated: per iteration the loss
    factor, whether the backward syncs, and whether a step follows it."""
    count, out = init_counts, []
    remainder = max_counts % n if max_counts is not None else None
    for _ in range(iters):
        if n == 1:
            factor = 1
        elif max_counts is None:
            factor = n
        else:
            factor = n if count < max_counts - remainder else remainder
        sync = (count + 1) % n == 0 or (max_counts is not None and count + 1 == max_counts)
        count += 1
        update = count % n == 0 or (max_counts is not None and count == max_counts)
        out.append((factor, sync, update))
    return out


def _net(seed=0):
    torch.manual_seed(seed)
    return nn.Sequential(nn.Linear(8, 16), nn.ReLU(), nn.Linear(16, 4), nn.Linear(4, 4))


def _wrapper(net, n, **kw):
    from embodiedscan_b200.engine import OptimWrapper
    ow = OptimWrapper(net, gc_interval=None, accumulative_counts=n, **kw)
    steps = []
    ow.optimizer.step = lambda: steps.append(ow.arena.grad.clone())     # the fused step is a CUDA kernel
    return ow, steps


def _run_schedule(ow, net, steps, iters):
    """Drive update_params as a training loop does and read back what the wrapper decided per iteration."""
    seen = []
    sync_at_backward = []
    p0 = ow.arena.params[0]
    h = p0.register_post_accumulate_grad_hook(lambda p: sync_at_backward.append(ow.reducer.sync))
    for i in range(iters):
        factor = 1 / float(ow.scale_loss(torch.tensor(1.0, dtype=torch.float64)))
        sync = ow.should_sync()
        n_before = len(steps)
        torch.manual_seed(i)
        ow.update_params(net(torch.randn(3, 8)).pow(2).sum())
        seen.append((round(factor), sync, len(steps) > n_before))
    h.remove()
    return seen, sync_at_backward


@pytest.mark.parametrize('n', [1, 2, 3, 4])
@pytest.mark.parametrize('status', [None, (0, 5), (0, 7), (3, 9)])
def test_schedule_matches_mmengine(n, status):
    net = _net()
    ow, steps = _wrapper(net, n)
    iters = 9
    if status is not None:
        init, mx = status
        with warnings.catch_warnings():
            warnings.simplefilter('ignore')
            ow.initialize_count_status(net, init, mx)
        iters = mx - init
        want = _mmengine_schedule(n, iters, init, mx)
    else:
        want = _mmengine_schedule(n, iters)
    got, sync_at_backward = _run_schedule(ow, net, steps, iters)
    assert got == want
    # the reducer saw the wrapper's decision while the backward ran, and is left ready to sync
    assert sync_at_backward == [w[1] for w in want] and ow.reducer.sync


def test_remainder_window_factors_and_steps():
    """max_counts=5, N=2: loss factors 2,2,2,2,1; steps after iterations 2, 4 and 5."""
    net = _net()
    ow, steps = _wrapper(net, 2)
    ow.initialize_count_status(nn.Linear(1, 1), 0, 5)
    got, _ = _run_schedule(ow, net, steps, 5)
    assert [g[0] for g in got] == [2, 2, 2, 2, 1]
    assert [i + 1 for i, g in enumerate(got) if g[2]] == [2, 4, 5]
    assert len(steps) == 3


def test_resume_inside_a_window_warns_and_finishes_it():
    net = _net()
    ow, steps = _wrapper(net, 2)
    with pytest.warns(UserWarning, match='not divisible'):
        ow.initialize_count_status(net, 3, 5)
    got, _ = _run_schedule(ow, net, steps, 2)
    assert got == [(2, True, True), (1, True, True)]
    with warnings.catch_warnings():
        warnings.simplefilter('error')
        ow.initialize_count_status(net, 4, 6)                 # divisible, no BatchNorm: silent
    with pytest.warns(UserWarning, match='BatchNorm'):
        ow.initialize_count_status(nn.Sequential(nn.BatchNorm1d(3)), 0, 6)


def test_accumulated_arena_is_the_sum_of_scaled_micro_batch_gradients():
    """Between the steps of a window nothing is zeroed: the arena after N micro-batches is the autograd sum of loss/N."""
    net, ref = _net(), _net()
    ow, steps = _wrapper(net, 3)
    for i in range(3):
        torch.manual_seed(i)
        x = torch.randn(3, 8)
        ow.update_params(net(x).pow(2).sum())
        (ref(x).pow(2).sum() / 3).backward()
    assert len(steps) == 1
    want = torch.zeros_like(steps[0])
    for p, o in zip(ow.arena.params, ow.arena.offsets):
        q = dict(zip([id(a) for a in net.parameters()], ref.parameters()))[id(p)]
        want[o:o + p.numel()] = q.grad.reshape(-1)
    assert torch.equal(steps[0], want)
    assert float(ow.arena.grad.abs().sum()) == 0, 'zero_grad runs once the window is complete'


def test_one_micro_batch_per_step_is_the_default():
    from embodiedscan_b200.engine import OptimWrapper
    net = _net()
    ow = OptimWrapper(net, gc_interval=None)
    assert ow.should_update() and ow.should_sync()
    loss = net(torch.randn(2, 8)).sum()
    assert ow.scale_loss(loss) is loss, 'N = 1 leaves the loss untouched (no extra op in the graph)'
    for bad in (0, -1, 1.5):
        with pytest.raises(ValueError):
            OptimWrapper(net, gc_interval=None, accumulative_counts=bad)


def test_optim_context_leaves_a_plain_model_alone_and_uses_no_sync():
    net = _net()
    ow, _ = _wrapper(net, 2)
    entered = []

    class WithNoSync(nn.Module):
        from contextlib import contextmanager

        @contextmanager
        def no_sync(self):
            entered.append(True)
            yield

    with ow.optim_context(net):
        pass
    with ow.optim_context(WithNoSync()):             # first micro-batch of a window: no sync
        pass
    assert entered == [True]
    ow._inner_count = 1
    with ow.optim_context(WithNoSync()):             # last micro-batch: sync
        pass
    assert entered == [True]


# ---- world 2 over gloo ------------------------------------------------------------------------------------------------
N_ACC = 2


def _batch(rank, i):
    torch.manual_seed(100 + 10 * rank + i)
    return torch.randn(5, 8)


def _worker(rank, world, port, q):
    sys.path.insert(0, ROOT)
    os.environ.update(MASTER_ADDR='127.0.0.1', MASTER_PORT=str(port))
    dist.init_process_group('gloo', rank=rank, world_size=world)
    from embodiedscan_b200.engine import OptimWrapper, broadcast_parameters
    torch.manual_seed(rank)
    net = torch.nn.Sequential(torch.nn.Linear(8, 16), torch.nn.ReLU(), torch.nn.Linear(16, 4), torch.nn.Linear(4, 4))
    ow = OptimWrapper(net, bucket_bytes=256, gc_interval=None, accumulative_counts=N_ACC)
    broadcast_parameters(ow.arena)
    calls = []
    real = dist.all_reduce

    def counting(*a, **k):
        calls.append(1)
        return real(*a, **k)
    dist.all_reduce = counting
    stepped = []
    ow.optimizer.step = lambda: stepped.append(ow.arena.grad.clone())
    per_micro_batch = []
    for i in range(N_ACC):
        out = net[2](net[1](net[0](_batch(rank, i))))            # net[3] unused: reduced by finish()
        ow.update_params(out.pow(2).sum())
        per_micro_batch.append(len(calls))
    dist.all_reduce = real
    # numpy copies travel by value (a shared-memory tensor needs its sender alive when the parent unpickles it)
    q.put((rank, ow.arena.flat.numpy().copy(), [g.numpy() for g in stepped], per_micro_batch, len(ow.arena.buckets),
           list(ow.reducer.pending) == list(ow.arena.n_params_in_bucket)))
    dist.destroy_process_group()


def test_gloo_world2_accumulation():
    import torch.multiprocessing as mp
    ctx = mp.get_context('spawn')
    q = ctx.Queue()
    port = 29500 + (os.getpid() + 700) % 2000
    procs = [ctx.Process(target=_worker, args=(r, 2, port, q)) for r in range(2)]
    for p in procs:
        p.start()
    res = sorted([q.get(timeout=120) for _ in range(2)], key=lambda t: t[0])
    for p in procs:
        p.join(30)
    (_, f0, s0, c0, nb, fresh0), (_, f1, s1, c1, _, fresh1) = res
    f0, f1 = torch.from_numpy(f0), torch.from_numpy(f1)
    s0, s1 = [torch.from_numpy(g) for g in s0], [torch.from_numpy(g) for g in s1]
    assert nb > 1, 'the test must exercise several buckets'
    assert c0[0] == c1[0] == 0, 'the first micro-batch of a window issues no collective'
    assert c0[1] == c1[1] == nb, 'the syncing micro-batch all-reduces every bucket once'
    assert len(s0) == len(s1) == 1 and torch.equal(s0[0], s1[0])
    assert fresh0 and fresh1, 'the reducer is reset for the next window'
    # single process: the sum over ranks and micro-batches of the gradients of loss / N
    sys.path.insert(0, ROOT)
    from embodiedscan_b200.engine import FlatArena
    torch.manual_seed(0)
    net = torch.nn.Sequential(torch.nn.Linear(8, 16), torch.nn.ReLU(), torch.nn.Linear(16, 4), torch.nn.Linear(4, 4))
    arena = FlatArena(net, bucket_bytes=256)
    assert torch.equal(arena.flat, f0) and torch.equal(f0, f1)
    for r in range(2):
        for i in range(N_ACC):
            (net[2](net[1](net[0](_batch(r, i)))).pow(2).sum() / N_ACC).backward()
    assert float(s0[0].abs().sum()) > 0
    assert torch.allclose(arena.grad, s0[0], rtol=1e-6, atol=1e-6)
