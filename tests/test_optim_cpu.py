"""CPU: engine.FusedAdamW as a torch Optimizer — mmengine's parameter-group layout, learning-rate schedulers writing the
groups, and state dicts that move between the arena optimiser and torch.optim.AdamW in both directions, bit for bit."""
import copy
import warnings

import pytest
import torch
import torch.nn as nn

LR, WD = 1e-3, 5e-4


def _mmengine_groups(model, base_lr, base_wd, paramwise_cfg):
    """Restatement of mmengine's DefaultOptimWrapperConstructor for `custom_keys`: without paramwise_cfg one group of
    model.parameters(); with it a recursive module walk, a module's own parameters before its children's, one group per
    parameter, frozen parameters appended as they are, keys tried longest first (alphabetical among equal lengths) against
    f'{prefix}.{name}'."""
    if not paramwise_cfg:
        return [{'params': list(model.parameters())}]
    keys = paramwise_cfg['custom_keys']
    order = sorted(sorted(keys), key=len, reverse=True)
    out = []

    def add(module, prefix):
        for name, p in module.named_parameters(recurse=False):
            g = {'params': [p]}
            if p.requires_grad:
                for k in order:
                    if k in f'{prefix}.{name}':
                        g['lr'] = base_lr * keys[k].get('lr_mult', 1.)
                        g['weight_decay'] = base_wd * keys[k].get('decay_mult', 1.)
                        break
            out.append(g)
        for cname, child in module.named_children():
            add(child, f'{prefix}.{cname}' if prefix else cname)
    add(model, '')
    return out


class _Net(nn.Module):
    def __init__(self):
        super().__init__()
        self.scale = nn.Parameter(torch.ones(3))
        self.decoder = nn.Sequential(nn.Linear(5, 7), nn.LayerNorm(7))
        self.text_encoder = nn.Linear(5, 3)
        self.text_encoder.requires_grad_(False)
        self.head = nn.ModuleDict(dict(cls=nn.Linear(7, 2), reg=nn.Linear(7, 4)))


PARAMWISE = dict(custom_keys={'decoder': dict(lr_mult=0.1, decay_mult=2.0), 'decoder.1': dict(lr_mult=0.0),
                              'head.cls': dict(decay_mult=0.0), 'head.reg': dict(lr_mult=3.0), 'text_encoder':
                              dict(lr_mult=0.0)})


def _net(seed=0):
    torch.manual_seed(seed)
    return _Net()


def _wrapper(model, paramwise_cfg=PARAMWISE):
    from embodiedscan_b200.engine import OptimWrapper
    return OptimWrapper(model, lr=LR, weight_decay=WD, paramwise_cfg=paramwise_cfg, gc_interval=None)


def _check_layout(ow, model, paramwise_cfg):
    want = _mmengine_groups(model, LR, WD, paramwise_cfg)
    got = ow.param_groups
    assert len(got) == len(want)
    for g, w in zip(got, want):
        assert len(g['params']) == len(w['params']) and all(a is b for a, b in zip(g['params'], w['params']))
        assert g['lr'] == w.get('lr', LR) and g['weight_decay'] == w.get('weight_decay', WD)


@pytest.mark.parametrize('paramwise', [False, True])
def test_groups_follow_mmengine_constructor(paramwise):
    from embodiedscan_b200.engine import FusedAdamW
    model = _net()
    cfg = PARAMWISE if paramwise else None
    ow = _wrapper(model, cfg)
    assert isinstance(ow.optimizer, torch.optim.Optimizer) and isinstance(ow.optimizer, FusedAdamW)
    _check_layout(ow, model, cfg)
    assert set(ow.param_groups[0]) == set(torch.optim.AdamW(model.parameters()).defaults) | {'params'}
    frozen = {id(p) for p in model.text_encoder.parameters()}
    assert not frozen & {id(p) for p in ow.arena.params}
    if not paramwise:
        assert ow.optimizer.group_of is None and ow.optimizer.lr_mult is None
        return
    # the kernel's group index: one slot per group that holds arena parameters, in group order
    slots = [k for k, g in enumerate(ow.param_groups) if id(g['params'][0]) not in frozen]
    assert ow.optimizer.group_of.dtype == torch.uint16
    gi = ow.optimizer.group_of.to(torch.int32)
    lm = ow.optimizer.lr_mult
    for p, o in zip(ow.arena.params, ow.arena.offsets):
        k = next(k for k, g in enumerate(ow.param_groups) if g['params'][0] is p)
        assert torch.all(gi[o:o + p.numel()] == slots.index(k))
        assert torch.allclose(lm[o:o + p.numel()], torch.tensor(ow.param_groups[k]['lr'] / LR))


def test_grounder_groups_follow_mmengine_constructor():
    """The grounding config's paramwise_cfg (configs/grounding/mv-grounding_8xb12_embodiedscan-vg-9dof.py): decoder at
    0.1 lr with decay_mult 1.0, text encoder at lr_mult 0 and frozen (requires_grad False)."""
    from embodiedscan_b200 import MODELS
    from embodiedscan_b200.synth import mv_grounding_config
    torch.manual_seed(0)
    model = MODELS.build(mv_grounding_config('C4-small'))
    cfg = dict(custom_keys={'text_encoder': dict(lr_mult=0.0), 'decoder': dict(lr_mult=0.1, decay_mult=1.0)})
    ow = _wrapper(model, cfg)
    _check_layout(ow, model, cfg)
    names = [n for n, _ in model.named_parameters()]
    assert len(ow.param_groups) == len(names)
    for n, g in zip(names, ow.param_groups):
        p = g['params'][0]
        if n.startswith('text_encoder'):
            assert not p.requires_grad and g['lr'] == LR          # frozen: in its group, no override, no arena slot
        elif 'decoder' in n and p.requires_grad:
            assert g['lr'] == LR * 0.1 and g['weight_decay'] == WD
    assert any('decoder' in n for n in names) and any(n.startswith('text_encoder') for n in names)


def _scheduled_lrs(opt, make, n=8):
    sched = make(opt)
    out = [[g['lr'] for g in opt.param_groups]]
    with warnings.catch_warnings():
        warnings.simplefilter('ignore')       # no optimizer.step() between scheduler steps: nothing to compute on the CPU
        for _ in range(n):
            sched.step()
            out.append([g['lr'] for g in opt.param_groups])
    return out


@pytest.mark.parametrize('kind', ['multistep', 'linear+multistep'])
def test_schedulers_attach_and_drive_groups(kind):
    from torch.optim import lr_scheduler as L
    from embodiedscan_b200.engine import param_groups

    def make(opt):
        if kind == 'multistep':
            return L.MultiStepLR(opt, milestones=[3, 6], gamma=0.1)
        return L.SequentialLR(opt, [L.LinearLR(opt, start_factor=0.1, total_iters=3),
                                    L.MultiStepLR(opt, milestones=[2, 4], gamma=0.1)], milestones=[3])
    model = _net()
    ow = _wrapper(model)
    twin = torch.optim.AdamW(param_groups(model, LR, WD, PARAMWISE), lr=LR, weight_decay=WD)
    ours, ref = _scheduled_lrs(ow.optimizer, make), _scheduled_lrs(twin, make)
    assert ours == ref
    assert ow.get_lr() == {'lr': ref[-1]}
    assert ow.get_momentum() == {'momentum': [0.9] * len(ref[-1])}
    assert all('initial_lr' in g for g in ow.param_groups)
    assert len(set(ours[0])) > 2 and ours[-1] != ours[0]


def _torch_twin(model, steps=3, seed=1, skip=()):
    """torch.optim.AdamW on the same groups, a few steps on random gradients (parameters named in `skip` get none)."""
    from embodiedscan_b200.engine import param_groups
    opt = torch.optim.AdamW(param_groups(model, LR, WD, PARAMWISE), lr=LR, weight_decay=WD)
    sched = torch.optim.lr_scheduler.MultiStepLR(opt, milestones=[2], gamma=0.1)
    g = torch.Generator().manual_seed(seed)
    for _ in range(steps):
        for n, p in model.named_parameters():
            p.grad = None if (not p.requires_grad or n in skip) else torch.randn(p.shape, generator=g)
        opt.step()
        sched.step()
    return opt


def _arena_moments(ow, p):
    o = ow.optimizer._offset[id(p)]
    return ow.optimizer.m[o:o + p.numel()].view_as(p), ow.optimizer.v[o:o + p.numel()].view_as(p)


def test_state_dict_round_trip_bitwise():
    model, twin_model = _net(), _net()
    twin = _torch_twin(twin_model)
    ow = _wrapper(model)
    ow.load_state_dict(copy.deepcopy(twin.state_dict()))
    assert ow.optimizer.step_count == 3
    assert ow.get_lr()['lr'] == [g['lr'] for g in twin.param_groups]
    assert [g['initial_lr'] for g in ow.param_groups] == [g['initial_lr'] for g in twin.param_groups]
    n_state = 0
    for p, q in zip(model.parameters(), twin_model.parameters()):
        if id(p) not in ow.optimizer._offset:
            continue
        m, v = _arena_moments(ow, p)
        assert torch.equal(m, twin.state[q]['exp_avg']) and torch.equal(v, twin.state[q]['exp_avg_sq'])
        n_state += 1
    assert n_state == len(ow.arena.params)

    # export, load into a fresh torch AdamW: the same tensors, the same groups
    sd = ow.state_dict()
    assert set(sd['state']) == {i for i, (n, p) in enumerate(model.named_parameters()) if p.requires_grad}
    fresh_model = _net()
    from embodiedscan_b200.engine import param_groups
    fresh = torch.optim.AdamW(param_groups(fresh_model, LR, WD, PARAMWISE), lr=LR, weight_decay=WD)
    fresh.load_state_dict(copy.deepcopy(sd))
    assert fresh.param_groups[0].keys() == twin.param_groups[0].keys()
    for a, b in zip(fresh.param_groups, twin.param_groups):
        assert {k: v for k, v in a.items() if k != 'params'} == {k: v for k, v in b.items() if k != 'params'}
    for p, q in zip(fresh_model.parameters(), twin_model.parameters()):
        if q in twin.state:
            for k in ('step', 'exp_avg', 'exp_avg_sq'):
                assert torch.equal(fresh.state[p][k], twin.state[q][k]), k
        else:
            assert p not in fresh.state


def test_missing_state_loads_zero_moments_under_the_shared_step():
    model, twin_model = _net(), _net()
    twin = _torch_twin(twin_model, skip=('head.reg.weight',))
    ow = _wrapper(model)
    ow.optimizer.m.fill_(7.)
    ow.optimizer.v.fill_(7.)
    ow.load_state_dict(twin.state_dict())
    m, v = _arena_moments(ow, model.head.reg.weight)
    assert not m.any() and not v.any()
    m, v = _arena_moments(ow, model.head.reg.bias)
    assert torch.equal(m, twin.state[twin_model.head.reg.bias]['exp_avg'])
    assert ow.optimizer.step_count == 3
    assert ow.optimizer.state_dict()['state'][
        [n for n, _ in model.named_parameters()].index('head.reg.weight')]['step'] == 3.


def test_load_rejects_mismatches_without_changing_state():
    from embodiedscan_b200.engine import param_groups
    twin_model = _net()
    good = _torch_twin(twin_model).state_dict()
    ow = _wrapper(_net())
    before = (ow.optimizer.m.clone(), ow.optimizer.step_count, [dict(g) for g in ow.param_groups])

    one_group = torch.optim.AdamW(twin_model.parameters(), lr=LR).state_dict()
    with pytest.raises(ValueError, match='parameter groups'):
        ow.load_state_dict(one_group)
    bad = copy.deepcopy(good)
    bad['param_groups'][2]['params'].append(999)
    with pytest.raises(ValueError, match='holds 2 parameters'):
        ow.load_state_dict(bad)
    bad = copy.deepcopy(good)
    bad['state'][1]['exp_avg'] = torch.zeros(3, 5)
    with pytest.raises(ValueError, match='shape'):
        ow.load_state_dict(bad)
    bad = copy.deepcopy(good)
    bad['state'][1]['step'] = torch.tensor(2.)
    with pytest.raises(ValueError, match='step count'):
        ow.load_state_dict(bad)
    bad = copy.deepcopy(good)
    bad['param_groups'][0]['amsgrad'] = True
    with pytest.raises(ValueError, match='amsgrad'):
        ow.load_state_dict(bad)
    assert torch.equal(ow.optimizer.m, before[0]) and ow.optimizer.step_count == before[1]
    assert [dict(g) for g in ow.param_groups] == before[2]
    # the one-group layout loads into the one-group wrapper
    ow1 = _wrapper(_net(), None)
    ow1.load_state_dict(torch.optim.AdamW(_net().parameters(), lr=LR).state_dict())
    assert ow1.optimizer.step_count == 0 and len(ow1.param_groups) == 1
    assert param_groups(_net(), LR, WD)[0]['params'].__len__() == len(list(_net().parameters()))


def test_zero_grad_keeps_gradients_in_the_arena():
    model = _net()
    ow = _wrapper(model)
    ow.arena.grad.fill_(1.)
    ow.optimizer.zero_grad()                     # torch's default would be set_to_none=True
    for p, o in zip(ow.arena.params, ow.arena.offsets):
        assert p.grad is not None and p.grad.data_ptr() == ow.arena.grad.data_ptr() + 4 * o
    assert not ow.arena.grad.any()
