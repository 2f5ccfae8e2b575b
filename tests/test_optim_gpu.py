"""GPU: the per-group fused AdamW step — the kernel per element against a float64 AdamW, whole trajectories under
learning-rate schedules against torch.optim.AdamW + clip_grad_norm_, hand-over of the state in both directions, and a
bit-exact resume of the deterministic bf16 detector step from a saved model + optimizer + scheduler checkpoint."""
import io

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu
DEV = 'cuda:0'
F32_EPS = 2.0 ** -23


def _close(a, b, rtol, what=''):
    a, b = a.detach().float().cpu(), b.detach().float().cpu()
    scale = max(float(b.abs().max()), 1e-6)
    err = float((a - b).abs().max())
    assert err <= rtol * scale, f'{what}: max abs err {err} vs scale {scale}'


def _adamw_launch(p, g, m, v, group_of, lr_wd, step, grad_scale, clip_state):
    from embodiedscan_b200 import _ffi
    lr_wd = torch.tensor(lr_wd, dtype=torch.float32)
    _ffi.call('esb_adamw_step_groups', p.data_ptr(), g.data_ptr(), m.data_ptr(), v.data_ptr(), _ffi.ptr(group_of),
              lr_wd.data_ptr(), lr_wd.numel() // 2, p.numel(), 0.9, 0.999, 1e-8, step, grad_scale,
              _ffi.ptr(clip_state), _ffi.stream())


@pytest.mark.parametrize('sizes,lrs,wds', [
    ([1001], [2e-3], [1e-2]),
    ([37, 1, 4099, 0, 515, 77777, 3], [1e-3, 5e-4, 0.0, 3e-3, 1e-4, 2e-3, 7e-4], [1e-4, 0.0, 5e-2, 1e-2, 0.3, 1e-3, 2e-2]),
])
def test_grouped_adamw_kernel_matches_float64(sizes, lrs, wds):
    """Several groups with their own lr and weight decay, one of them at lr 0, odd sizes: every element within a few float32
    ulps of AdamW in float64 on the same float32 inputs; the lr-0 slice and its moments bit-unchanged."""
    from embodiedscan_b200 import _ffi
    gen = torch.Generator().manual_seed(5)
    n = sum(sizes)
    p0 = torch.randn(n, generator=gen)
    g0 = torch.randn(n, generator=gen) * 3
    m0 = torch.randn(n, generator=gen) * 0.1
    v0 = torch.rand(n, generator=gen) * 0.05
    grp = torch.cat([torch.full((s, ), k, dtype=torch.int32) for k, s in enumerate(sizes)])
    p, g, m, v = (t.to(DEV) for t in (p0, g0, m0, v0))
    group_of = grp.numpy().astype(np.uint16)
    group_of = torch.from_numpy(group_of).to(DEV) if len(sizes) > 1 else None
    clip = torch.zeros(3, device=DEV)
    _ffi.call('esb_grad_clip_coef', g.data_ptr(), n, 5.0, 0.5, clip.data_ptr(), _ffi.stream())
    step = 1        # 1 - beta**1 is exact in float32: the kernel's bias corrections equal the reference's (later steps: below)
    lr_wd = [x for pair in zip(lrs, wds) for x in pair]
    _adamw_launch(p, g, m, v, group_of, lr_wd, step, 0.5, clip)
    coef = float(clip[2])
    assert 0 < coef < 1, 'the clip must be active'

    d = torch.float64
    lr = torch.tensor(lrs, dtype=torch.float32).to(d)[grp.long()]
    wd = torch.tensor(wds, dtype=torch.float32).to(d)[grp.long()]
    b1, b2, eps = np.float32(0.9).item(), np.float32(0.999).item(), np.float32(1e-8).item()
    bc1, bc2_sqrt = 1 - b1 ** step, float(np.sqrt(np.float32(1 - b2 ** step)))      # float32 scalars, as the kernel's
    gi = g0.to(d) * (0.5 * coef)
    m_ref = b1 * m0.to(d) + (1 - b1) * gi
    v_ref = b2 * v0.to(d) + (1 - b2) * gi * gi
    decayed = p0.to(d) * (1 - lr * wd)
    upd = lr / bc1 * m_ref / (v_ref.sqrt() / bc2_sqrt + eps)
    p_ref = decayed - upd
    frozen = lr == 0
    live = ~frozen
    for got, ref, mag, what in ((m, m_ref, b1 * m0.to(d).abs() + (1 - b1) * gi.abs(), 'exp_avg'),
                                (v, v_ref, v_ref.abs(), 'exp_avg_sq'),
                                (p, p_ref, decayed.abs() + upd.abs(), 'param')):
        err = (got.cpu().to(d) - ref).abs()[live]
        bound = 8 * F32_EPS * mag[live] + 1e-30
        assert bool((err <= bound).all()), f'{what}: worst {float((err / bound).max()):.2f} of the bound'
    for got, before in ((p, p0), (m, m0), (v, v0)):
        assert torch.equal(got.cpu()[frozen], before[frozen])
    assert frozen.any() == (0.0 in lrs)


def test_group_table_limits_are_errors():
    x = torch.zeros(64, device=DEV)
    idx = torch.from_numpy(np.zeros(64, dtype=np.uint16)).to(DEV)
    with pytest.raises(RuntimeError, match='groups'):
        _adamw_launch(x, x, x, x, idx, [1e-3, 0.] * 2049, 1, 1.0, None)
    with pytest.raises(RuntimeError, match='group_of'):
        _adamw_launch(x, x, x, x, None, [1e-3, 0.] * 2, 1, 1.0, None)
    with pytest.raises(RuntimeError, match='group_of'):
        _adamw_launch(x, x, x, x, idx, [1e-3, 0.], 1, 1.0, None)


PARAMWISE = dict(custom_keys={'0.': dict(lr_mult=2.0, decay_mult=0.0), '2.bias': dict(lr_mult=0.5, decay_mult=3.0),
                              '4.': dict(lr_mult=0.0)})
LR, WD, MAX_NORM = 1e-3, 1e-2, 0.5


def _nets(seed=7):
    torch.manual_seed(seed)

    def make():
        return torch.nn.Sequential(torch.nn.Linear(37, 53), torch.nn.ReLU(), torch.nn.Linear(53, 29), torch.nn.ReLU(),
                                   torch.nn.Linear(29, 11)).to(DEV)
    net, ref = make(), make()
    ref.load_state_dict(net.state_dict())
    return net, ref


def _schedule(opt):
    L = torch.optim.lr_scheduler
    return L.SequentialLR(opt, [L.LinearLR(opt, start_factor=0.25, total_iters=2),
                                L.MultiStepLR(opt, milestones=[2], gamma=0.1)], milestones=[2])


def _torch_step(ref, opt, x):
    (ref(x) ** 2).sum().backward()
    torch.nn.utils.clip_grad_norm_(ref.parameters(), MAX_NORM)
    opt.step()
    opt.zero_grad()


def _compare(net, ow, ref, opt):
    for (name, a), b in zip(net.named_parameters(), ref.parameters()):
        _close(a, b, 1e-5, f'{name} parameters')
        k = next(k for k, g in enumerate(ow.param_groups) if any(p is a for p in g['params']))
        if ow.param_groups[k]['lr'] == 0:        # torch AdamW still updates the moments of an lr-0 group; the arena keeps them
            continue
        o = ow.optimizer._offset[id(a)]
        _close(ow.optimizer.m[o:o + a.numel()], opt.state[b]['exp_avg'].reshape(-1), 1e-5, f'{name} exp_avg')
        # the kernel forms 1 - beta2 from the float32 beta2 (0.99998713e-3), torch from the double (1.00000005e-3 once
        # rounded): each step's new term of exp_avg_sq differs by 1.29e-5 relative, so that moment gets 2e-5
        _close(ow.optimizer.v[o:o + a.numel()], opt.state[b]['exp_avg_sq'].reshape(-1), 2e-5, f'{name} exp_avg_sq')


def test_scheduled_paramwise_trajectory_matches_torch():
    """7 steps: LinearLR warm-up, then MultiStepLR crossing its milestone; clipping active; lr_mult / decay_mult per group.
    Both optimisers see the same gradients (torch's, copied into the arena), so what differs is the optimiser alone."""
    from embodiedscan_b200.engine import OptimWrapper, param_groups
    net, ref = _nets()
    ow = OptimWrapper(net, lr=LR, weight_decay=WD, max_norm=MAX_NORM, paramwise_cfg=PARAMWISE, gc_interval=None)
    opt = torch.optim.AdamW(param_groups(ref, LR, WD, PARAMWISE), lr=LR, weight_decay=WD)
    s_ours, s_ref = _schedule(ow.optimizer), _schedule(opt)
    lrs, norms = [], []
    for _ in range(7):
        x = torch.randn(64, 37, device=DEV)
        (ref(x) ** 2).sum().backward()
        for p, q in zip(net.parameters(), ref.parameters()):
            p.grad.copy_(q.grad)
        torch.nn.utils.clip_grad_norm_(ref.parameters(), MAX_NORM)
        opt.step()
        opt.zero_grad()
        ow.step()
        ow.zero_grad()
        norms.append(float(ow.optimizer.grad_norm))
        s_ours.step()
        s_ref.step()
        lrs.append(ow.get_lr()['lr'])
        assert lrs[-1] == [g['lr'] for g in opt.param_groups]
    assert len({l[1] for l in lrs}) >= 3 and max(norms) > MAX_NORM, (lrs, norms)
    _compare(net, ow, ref, opt)


@pytest.mark.parametrize('direction', ['torch_to_arena', 'arena_to_torch'])
def test_hand_over_mid_run(direction):
    from embodiedscan_b200.engine import OptimWrapper, param_groups
    net, ref = _nets()
    ow = OptimWrapper(net, lr=LR, weight_decay=WD, max_norm=MAX_NORM, paramwise_cfg=PARAMWISE, gc_interval=None)
    opt = torch.optim.AdamW(param_groups(ref, LR, WD, PARAMWISE), lr=LR, weight_decay=WD)
    xs = [torch.randn(64, 37, device=DEV) for _ in range(6)]
    for x in xs[:3]:
        if direction == 'torch_to_arena':
            _torch_step(ref, opt, x)
        else:
            ow.update_params((net(x) ** 2).sum())
    buf = io.BytesIO()
    if direction == 'torch_to_arena':
        torch.save(dict(model=ref.state_dict(), optimizer=opt.state_dict()), buf)
        buf.seek(0)
        ck = torch.load(buf)
        net.load_state_dict(ck['model'])
        ow.load_state_dict(ck['optimizer'])
        assert ow.optimizer.step_count == 3
    else:
        torch.save(dict(model=net.state_dict(), optimizer=ow.state_dict()), buf)
        buf.seek(0)
        ck = torch.load(buf)
        ref.load_state_dict(ck['model'])
        opt.load_state_dict(ck['optimizer'])
        # the lr-0 group: torch starts from the arena's (untouched, zero) moments
    for x in xs[3:]:
        _torch_step(ref, opt, x)
        ow.update_params((net(x) ** 2).sum())
    _compare(net, ow, ref, opt)


def test_bf16_detector_resume_is_bit_exact():
    """Run A: 4 train steps. Run B: 2 steps, checkpoint (model, optimizer, scheduler) through torch.save, a fresh model and
    wrapper restored in mmengine's resume order (weights, optimizer, scheduler), 2 more steps. The deterministic bf16 step
    makes every parameter, buffer, moment and the last two losses bit-identical."""
    from embodiedscan_b200 import MODELS
    from embodiedscan_b200.engine import OptimWrapper
    from embodiedscan_b200.synth import mv_det3d_config, synth_batch
    cfg = dict(mv_det3d_config('C2'), compute_dtype=torch.bfloat16)

    def build(seed):
        torch.manual_seed(seed)
        model = MODELS.build(cfg).to(DEV).train()
        ow = OptimWrapper(model, lr=1e-3, weight_decay=1e-4, gc_interval=None)
        sched = torch.optim.lr_scheduler.MultiStepLR(ow.optimizer, milestones=[1, 3], gamma=0.1)
        return model, ow, sched

    def step(model, ow, sched, i):
        torch.manual_seed(100 + i)
        batch = synth_batch(1, 2, n_views=2, H=240, W=320, n_points=2000, augment=True)
        logs = model.train_step(dict(inputs=batch['inputs'], data_samples=batch['data_samples']), ow)
        sched.step()
        return float(logs['loss'])

    a = build(0)
    loss_a = [step(*a, i) for i in range(4)]
    b = build(0)
    loss_b = [step(*b, i) for i in range(2)]
    buf = io.BytesIO()
    torch.save(dict(model=b[0].state_dict(), optimizer=b[1].state_dict(), scheduler=b[2].state_dict()), buf)
    del b
    buf.seek(0)
    ck = torch.load(buf)
    c = build(1)
    c[0].load_state_dict(ck['model'])
    c[1].load_state_dict(ck['optimizer'])
    c[2].load_state_dict(ck['scheduler'])
    assert c[1].get_lr() == {'lr': [ck['optimizer']['param_groups'][0]['lr']]} and c[1].optimizer.step_count == 2
    loss_b += [step(*c, i) for i in range(2, 4)]
    assert loss_a[2:] == loss_b[2:], (loss_a, loss_b)
    assert a[1].optimizer.step_count == c[1].optimizer.step_count == 4
    for (name, x), y in zip(a[0].named_parameters(), c[0].parameters()):
        assert torch.equal(x, y), name
    for (name, x), y in zip(a[0].named_buffers(), c[0].buffers()):
        assert torch.equal(x, y), name
    assert torch.equal(a[1].optimizer.m, c[1].optimizer.m) and torch.equal(a[1].optimizer.v, c[1].optimizer.v)
    assert torch.equal(a[1].arena.bf16, c[1].arena.bf16)
