"""GPU: gradient accumulation over micro-batches (engine.OptimWrapper `accumulative_counts`).

- The kernels that write gradient slots in place (sparse BatchNorm backward in direct mode, the `_slot` sparse wgrads) add
  one pass's finished sum to whatever the slot holds with one rounded add, and compute everything else from that pass
  alone.
- Two micro-batches on the arena give every parameter the bits plain autograd gives it (`grad += fresh`).
- Accumulated bf16 training is deterministic, N = 1 is today's step, and a small net follows torch's
  loss / N -> backward x N -> clip_grad_norm_ -> AdamW trajectory, remainder window included.
- Two GPUs over NCCL: a non-syncing micro-batch launches no bucket, and the window's arena is the sum over ranks and
  micro-batches (skipped on one GPU)."""
import os
import sys

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
pytestmark = pytest.mark.gpu
DEV = 'cuda:0'


# ---- kernels -----------------------------------------------------------------------------------------------------------
def _norm_bwd(x, y, dy, mean, rstd, gamma, sg, sgx, zero_sums):
    from embodiedscan_b200 import _ffi
    N, C = x.shape
    dx, dres = torch.empty_like(x), torch.empty_like(x)
    _ffi.call('esb_norm_bwd', x.data_ptr(), y.data_ptr(), dy.data_ptr(), None, None, 1, N, N, C, mean.data_ptr(),
              rstd.data_ptr(), gamma.data_ptr(), 1, sg.data_ptr(), sgx.data_ptr(), dx.data_ptr(), dres.data_ptr(),
              zero_sums, _ffi.dtype_code(x.dtype), _ffi.stream())
    return dx, dres


@pytest.mark.parametrize('dtype', [torch.float32, torch.bfloat16])
@pytest.mark.parametrize('N,C', [(3000, 64), (777, 13), (1, 24), (5000, 200)])
def test_norm_bwd_direct_mode_adds_this_pass_sums_to_the_slots(dtype, N, C):
    """S = 1 (BatchNorm). dx / dres with slots already holding earlier gradients are bit-equal to a run on zeroed slots and
    to the plain (zero_sums = 1) run; each slot becomes prev + this pass's sums, one float32 add."""
    g = torch.Generator(device=DEV).manual_seed(N * 1000 + C)
    x = (torch.randn(N, C, device=DEV, generator=g) * 2 + 0.5).to(dtype)
    y = torch.relu(torch.randn(N, C, device=DEV, generator=g)).to(dtype)        # ReLU output: act = 1 reads it
    dy = torch.randn(N, C, device=DEV, generator=g).to(dtype)
    mean = x.float().mean(0, keepdim=True).contiguous()
    rstd = torch.rsqrt(x.float().var(0, unbiased=False, keepdim=True) + 1e-5).contiguous()
    gamma = torch.randn(C, device=DEV, generator=g)
    sg, sgx = torch.empty(C, device=DEV), torch.empty(C, device=DEV)
    dx0, dres0 = _norm_bwd(x, y, dy, mean, rstd, gamma, sg, sgx, 1)
    zg, zgx = torch.zeros(C, device=DEV), torch.zeros(C, device=DEV)
    dx1, dres1 = _norm_bwd(x, y, dy, mean, rstd, gamma, zg, zgx, 0)
    prev_g = torch.randn(C, device=DEV, generator=g) * 100
    prev_gx = torch.randn(C, device=DEV, generator=g) * 1e-3
    slot_g, slot_gx = prev_g.clone(), prev_gx.clone()
    dx2, dres2 = _norm_bwd(x, y, dy, mean, rstd, gamma, slot_g, slot_gx, 0)
    torch.cuda.synchronize()
    assert torch.equal(dx1, dx0) and torch.equal(dres1, dres0)
    assert torch.equal(dx2, dx0) and torch.equal(dres2, dres0), 'dx must come from this pass\'s sums alone'
    assert torch.equal(zg, sg) and torch.equal(zgx, sgx), 'a zeroed slot receives the sums bit for bit'
    assert torch.equal(slot_g, prev_g + sg) and torch.equal(slot_gx, prev_gx + sgx)
    assert bool((sg != 0).any())


def _pairs(n, K):
    """K offsets, each pairing every input row with a shuffled output row (pair lists grouped by offset)."""
    g = torch.Generator().manual_seed(n + K)
    pin = torch.cat([torch.randperm(n, generator=g) for _ in range(K)]).int()
    pout = torch.cat([torch.randperm(n, generator=g) for _ in range(K)]).int()
    koff = torch.arange(0, (K + 1) * n, n, dtype=torch.int32)
    return pin.to(DEV), pout.to(DEV), koff.to(DEV)


@pytest.mark.parametrize('kind,dtype,cin,cout,K', [('tc', torch.bfloat16, 64, 128, 3), ('tc', torch.bfloat16, 128, 64, 1),
                                                    ('simt', torch.bfloat16, 32, 24, 3), ('simt', torch.float32, 16, 13, 2)])
def test_sparse_wgrad_slot_adds_its_finished_sum_to_the_slot(kind, dtype, cin, cout, K):
    """esb_spconv_{tc_,}wgrad_slot: into a non-zero slot, prev + the gradient computed into zeros (one float32 add); into
    zeros, the bits of the plain entry point."""
    from embodiedscan_b200 import _ffi
    n = 20000
    g = torch.Generator(device=DEV).manual_seed(cin + cout)
    x = torch.randn(n, cin, device=DEV, generator=g).to(dtype)
    dy = torch.randn(n, cout, device=DEV, generator=g).to(dtype)
    pin, pout, koff = _pairs(n, K)

    def wgrad(dw, slot='_slot'):
        if kind == 'tc':
            _ffi.call('esb_spconv_tc_wgrad' + slot, x.data_ptr(), dy.data_ptr(), pin.data_ptr(), pout.data_ptr(), koff.data_ptr(),
                      dw.data_ptr(), K * n, cin, cout, K, _ffi.stream())
        else:
            _ffi.call('esb_spconv_wgrad' + slot, x.data_ptr(), dy.data_ptr(), pin.data_ptr(), pout.data_ptr(), koff.data_ptr(),
                      dw.data_ptr(), K * n, cin, cout, K, _ffi.dtype_code(dtype), _ffi.stream())
        return dw

    fresh = wgrad(torch.zeros(K, cin, cout, device=DEV))
    prev = torch.randn(K, cin, cout, device=DEV, generator=g) * 50
    slot = wgrad(prev.clone())
    plain = wgrad(torch.zeros(K, cin, cout, device=DEV), '')
    torch.cuda.synchronize()
    assert torch.equal(fresh, plain) and bool((fresh != 0).any())
    assert torch.equal(slot, prev + fresh)
    assert not bool(torch.signbit(fresh[fresh == 0]).any()), 'a sum from +0 is never -0'


# ---- models ------------------------------------------------------------------------------------------------------------
def _batch(i, n_scans=2):
    from embodiedscan_b200.synth import synth_batch
    return synth_batch(10 + i, n_scans, n_views=2, H=240, W=320, n_points=2000, augment=True)


@pytest.mark.parametrize('variant,dtype', [('C1', torch.bfloat16), ('C2', torch.bfloat16), ('C1', torch.float32)])
def test_two_micro_batches_on_the_arena_equal_plain_autograd(variant, dtype):
    """Two forward + backward passes without zero_grad: the arena (direct sparse wgrad / BatchNorm slots, bf16 shadow
    operands, graphed 2D branch) against two plain-autograd twins. bf16: every gradient bit-equal. fp32: the bounds of
    test_model_gpu's one-pass check (the 2D branch's fp32 atomics differ run to run)."""
    from embodiedscan_b200 import MODELS
    from embodiedscan_b200.engine import FlatArena
    from embodiedscan_b200.synth import mv_det3d_config
    torch.manual_seed(0)
    cfg = dict(mv_det3d_config(variant), compute_dtype=dtype)
    models = [MODELS.build(cfg).to(DEV).train() for _ in range(3)]
    for m in models[1:]:
        m.load_state_dict(models[0].state_dict())
    for m in models[:2]:     # plain autograd: `grad += fresh` from the first pass on
        for p in m.parameters():
            if p.requires_grad:
                p.grad = torch.zeros_like(p)
    arena = FlatArena(models[2])
    arena.zero_grad()
    batches = [_batch(0), _batch(1)]
    for m in models:
        for b in batches:
            data = m.data_preprocessor(dict(inputs=b['inputs'], data_samples=b['data_samples']), True)
            sum(m(**data, mode='loss').values()).backward()
    torch.cuda.synchronize()
    if dtype == torch.float32:
        num = den = 0.
        for (name, p0), p2 in zip(models[0].named_parameters(), models[2].parameters()):
            if not p0.requires_grad:
                continue
            num += float((p0.grad - p2.grad).norm()) ** 2
            den += float(p0.grad.norm()) ** 2
            scale = max(float(p0.grad.abs().max()), 1e-8)
            assert float((p0.grad - p2.grad).abs().max()) / scale <= 2e-3, name
        assert (num / max(den, 1e-30)) ** 0.5 <= 1e-3
        return
    differ = []
    for (name, p0), p1, p2 in zip(models[0].named_parameters(), models[1].parameters(), models[2].parameters()):
        if not p0.requires_grad:
            continue
        assert torch.equal(p0.grad, p1.grad), f'{name}: two plain runs differ'
        if not torch.equal(p0.grad, p2.grad):
            differ.append(name)
    assert not differ, f'accumulated arena gradients differ from autograd: {differ}'
    assert sum(bool(p.grad.any()) for p in models[2].parameters() if p.requires_grad) > 10


def _train(n_acc, steps, seed=0, pass_counts=True):
    from embodiedscan_b200 import MODELS
    from embodiedscan_b200.engine import OptimWrapper
    from embodiedscan_b200.synth import mv_det3d_config
    cfg = dict(mv_det3d_config('C2'), compute_dtype=torch.bfloat16)
    torch.manual_seed(seed)
    model = MODELS.build(cfg).to(DEV).train()
    kw = dict(accumulative_counts=n_acc) if pass_counts else {}
    ow = OptimWrapper(model, lr=1e-3, weight_decay=1e-4, gc_interval=None, **kw)
    losses = []
    for i in range(steps * n_acc):
        b = _batch(i, 1)
        losses.append(float(model.train_step(dict(inputs=b['inputs'], data_samples=b['data_samples']), ow)['loss']))
    torch.cuda.synchronize()
    return model, ow, losses


def test_accumulated_bf16_training_is_deterministic():
    a = _train(2, 3)
    b = _train(2, 3)
    assert a[1].optimizer.step_count == b[1].optimizer.step_count == 3
    assert a[2] == b[2]
    assert torch.equal(a[1].arena.flat, b[1].arena.flat)
    assert torch.equal(a[1].optimizer.m, b[1].optimizer.m) and torch.equal(a[1].optimizer.v, b[1].optimizer.v)
    for (name, x), y in zip(a[0].named_buffers(), b[0].buffers()):
        assert torch.equal(x, y), name


def test_one_micro_batch_per_step_keeps_the_bits():
    a = _train(1, 3, pass_counts=False)
    b = _train(1, 3)
    assert a[2] == b[2]
    assert torch.equal(a[1].arena.flat, b[1].arena.flat)
    assert torch.equal(a[1].optimizer.m, b[1].optimizer.m) and torch.equal(a[1].optimizer.v, b[1].optimizer.v)


LR, WD, MAX_NORM = 1e-3, 1e-2, 0.5


def test_trajectory_matches_torch_with_a_remainder_window():
    """accumulative_counts=3 over 7 iterations (windows of 3, 3, 1): torch runs loss / factor -> backward per micro-batch,
    clip_grad_norm_ and AdamW per window. Parameters and moments within test_optim_gpu's bounds."""
    from embodiedscan_b200.engine import OptimWrapper
    torch.manual_seed(7)

    def make():
        return torch.nn.Sequential(torch.nn.Linear(37, 53), torch.nn.ReLU(), torch.nn.Linear(53, 29), torch.nn.ReLU(),
                                   torch.nn.Linear(29, 11)).to(DEV)
    net, ref = make(), make()
    ref.load_state_dict(net.state_dict())
    ow = OptimWrapper(net, lr=LR, weight_decay=WD, max_norm=MAX_NORM, gc_interval=None, accumulative_counts=3)
    ow.initialize_count_status(net, 0, 7)
    opt = torch.optim.AdamW(ref.parameters(), lr=LR, weight_decay=WD)
    factors, norms = [3, 3, 3, 3, 3, 3, 1], []
    for i in range(7):
        x = torch.randn(64, 37, device=DEV)
        ow.update_params((net(x) ** 2).sum())
        ((ref(x) ** 2).sum() / factors[i]).backward()
        if i in (2, 5, 6):
            norms.append(float(torch.nn.utils.clip_grad_norm_(ref.parameters(), MAX_NORM)))
            opt.step()
            opt.zero_grad()
            assert ow.optimizer.step_count == len(norms)
            assert abs(float(ow.optimizer.grad_norm) - norms[-1]) <= 1e-5 * norms[-1]
    assert max(norms) > MAX_NORM, norms
    for (name, a), b in zip(net.named_parameters(), ref.parameters()):
        for got, want, tol, what in ((a, b, 1e-5, 'param'),
                                     (ow.optimizer.m[ow.optimizer._offset[id(a)]:][:a.numel()], opt.state[b]['exp_avg'],
                                      1e-5, 'exp_avg'),
                                     (ow.optimizer.v[ow.optimizer._offset[id(a)]:][:a.numel()], opt.state[b]['exp_avg_sq'],
                                      2e-5, 'exp_avg_sq')):
            got, want = got.detach().float().reshape(-1).cpu(), want.detach().float().reshape(-1).cpu()
            scale = max(float(want.abs().max()), 1e-6)
            assert float((got - want).abs().max()) <= tol * scale, f'{name} {what}'


# ---- two GPUs over NCCL ------------------------------------------------------------------------------------------------
def _worker(rank, world, port, q):
    sys.path.insert(0, ROOT)
    import torch.distributed as dist
    os.environ.update(MASTER_ADDR='127.0.0.1', MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world))
    torch.cuda.set_device(rank)
    dev = torch.device('cuda', rank)
    dist.init_process_group('nccl', rank=rank, world_size=world, device_id=dev)
    from embodiedscan_b200 import MODELS
    from embodiedscan_b200.engine import OptimWrapper, broadcast_parameters
    from embodiedscan_b200.synth import mv_det3d_config, synth_batch
    torch.manual_seed(0)
    model = MODELS.build(mv_det3d_config('C1')).to(dev).train()
    model.overlap_2d_3d = True
    for m in model.modules():                 # running statistics must not drift between the passes below
        if isinstance(m, torch.nn.modules.batchnorm._BatchNorm):
            m.momentum = 0.0
    n_acc = 2
    ow = OptimWrapper(model, bucket_bytes=1 << 20, gc_interval=None, accumulative_counts=n_acc)
    broadcast_parameters(ow.arena)
    arena, red = ow.arena, ow.reducer
    batches = [[synth_batch(20 + 2 * r + i, 1, n_views=2, H=240, W=320, n_points=2000, device=dev) for i in range(n_acc)]
               for r in range(world)]
    head, n_pos = model.bbox_head, {}
    orig_reduce = head._reduce_mean
    launches = []
    orig_launch = red._launch
    red._launch = lambda b: (launches.append(b), orig_launch(b))
    window = []
    ow.optimizer.step = lambda: window.append(arena.grad.clone())

    # the head normalises by the mean over ranks of the positives of each micro-batch: the single-rank passes below use
    # the normaliser of the distributed pass of the same micro-batch
    def recording(x, i):
        n_pos[i] = orig_reduce(x).clone()
        return n_pos[i]
    per_micro_batch = []
    for i, b in enumerate(batches[rank]):
        head._reduce_mean = lambda x, i=i: recording(x, i)
        data = model.data_preprocessor(dict(inputs=b['inputs'], data_samples=b['data_samples']), True)
        ow.update_params(sum(model(**data, mode='loss').values()))
        torch.cuda.synchronize()
        per_micro_batch.append(len(launches))
    singles = []
    red.enabled = False
    for r in range(world):
        for i, b in enumerate(batches[r]):
            head._reduce_mean = lambda x, i=i: n_pos[i].clone()
            arena.zero_grad()
            red.reset()
            data = model.data_preprocessor(dict(inputs=b['inputs'], data_samples=b['data_samples']), True)
            (sum(model(**data, mode='loss').values()) / n_acc).backward()
            torch.cuda.synchronize()
            singles.append(arena.grad.clone())
    want = sum(singles)
    scale = float(want.abs().max())
    err = float((window[0] - want).abs().max())
    q.put((rank, per_micro_batch, len(arena.buckets), err, scale))
    dist.destroy_process_group()


@pytest.mark.skipif(not torch.cuda.is_available() or torch.cuda.device_count() < 2, reason='needs 2 GPUs')
def test_nccl_accumulated_window_equals_sum_of_single_rank_micro_batches():
    import torch.multiprocessing as mp
    ctx = mp.get_context('spawn')
    q = ctx.Queue()
    port = 29500 + (os.getpid() + 1100) % 2000
    procs = [ctx.Process(target=_worker, args=(r, 2, port, q)) for r in range(2)]
    for p in procs:
        p.start()
    res = sorted([q.get(timeout=600) for _ in range(2)])
    for p in procs:
        p.join(60)
    for rank, per_micro_batch, n_buckets, err, scale in res:
        assert per_micro_batch[0] == 0, (rank, 'the non-syncing micro-batch launched a bucket')
        assert per_micro_batch[1] == n_buckets > 3, (rank, per_micro_batch, n_buckets)
        assert scale > 0 and err <= 1e-4 * scale, (rank, err, scale)
