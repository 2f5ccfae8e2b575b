"""Training-step runtime for the hot path: flat parameter/gradient arenas, fused clip + AdamW kernels, and data-parallel
gradient all-reduce over NCCL (NVLink 5 / NVSwitch) launched per bucket as soon as a bucket's gradients are complete.

Replaces, for this path, mmengine's OptimWrapper + MMDistributedDataParallel (†upstream; optimizer and clip settings at
configs/detection/mv-det3d_8xb4_embodiedscan-3d-284class-9dof.py:219-223): one process per GPU, scans sharded across
ranks, the only bulk collective is the gradient SUM (averaged inside the AdamW kernel), no host synchronisation.
"""
from contextlib import contextmanager
from typing import List, Optional

import numpy as np
import torch
import torch.distributed as dist
import torch.nn as nn

from ._ffi import call, ptr, stream


ALIGN = 16   # elements

# CUDA streams other than the default one on which kernels write gradients into the arena (the detector's 2D side stream
# registers itself here): a bucket's all-reduce must be ordered after ALL of them, not just the stream its last hook ran on.
GRAD_STREAMS = set()


def register_grad_stream(s):
    GRAD_STREAMS.add(s)


class FlatArena:
    """All trainable parameters live in ONE contiguous fp32 buffer, their gradients in another (same offsets)."""

    def __init__(self, model: nn.Module, bucket_bytes: int = 64 << 20):
        params = [p for p in model.parameters() if p.requires_grad]
        # reverse registration order ~ the order autograd finishes gradients, so buckets complete front to back
        params = params[::-1]
        self.params = params
        dev = params[0].device
        offs, n = [], 0
        for p in params:
            offs.append(n)
            n += (p.numel() + ALIGN - 1) // ALIGN * ALIGN     # 64 B in fp32, 32 B in the bf16 shadow (16 B cp.async loads)
        self.numel = n
        self.flat = torch.zeros(n, dtype=torch.float32, device=dev)
        self.grad = torch.zeros(n, dtype=torch.float32, device=dev)
        self.offsets = offs
        self.bf16 = torch.zeros(n, dtype=torch.bfloat16, device=dev) if dev.type == 'cuda' else None
        for p, o in zip(params, offs):
            self.flat[o:o + p.numel()].copy_(p.data.reshape(-1).float())
            p.data = self.flat[o:o + p.numel()].view_as(p)
            p.grad = self.grad[o:o + p.numel()].view_as(p)
            if self.bf16 is not None:
                p._esb_bf16 = self.bf16[o:o + p.numel()].view_as(p)     # bf16 operand copy, refreshed once per step
                p._esb_grad_direct = True                                # kernels may accumulate into p.grad in place
        self.refresh_bf16()
        # buckets: contiguous [start, end) ranges of ~bucket_bytes
        self.buckets, self.bucket_of = [], []
        start, cur = 0, 0
        per = max(bucket_bytes // 4, 1)
        for i, (p, o) in enumerate(zip(params, offs)):
            end = o + (p.numel() + ALIGN - 1) // ALIGN * ALIGN
            self.bucket_of.append(len(self.buckets))
            if end - start >= per or i == len(params) - 1:
                self.buckets.append((start, end))
                start = end
        self.n_params_in_bucket = [0] * len(self.buckets)
        for b in self.bucket_of:
            self.n_params_in_bucket[b] += 1

    def refresh_bf16(self):
        """fp32 master arena -> bf16 compute copy: ONE launch for the whole model."""
        if self.bf16 is not None:
            call('esb_cast_f32_to_bf16', ptr(self.flat), ptr(self.bf16), self.numel, stream())
            for p in self.params:            # consumers use the shadow only while the parameter is unchanged since now
                p._esb_bf16_version = p._version

    def zero_grad(self):
        self.grad.zero_()
        for p, o in zip(self.params, self.offsets):  # autograd may have replaced .grad; re-point it at the arena
            p._esb_uses = p._esb_pass_uses = 0
            if p.grad is None or p.grad.data_ptr() != self.grad.data_ptr() + 4 * o:
                p.grad = self.grad[o:o + p.numel()].view_as(p)


class DataParallelReducer:
    """Per-bucket asynchronous all-reduce(SUM) of the gradient arena, overlapped with the rest of backward.

    With gradient accumulation only the last backward pass of a window reduces: `sync` (set by OptimWrapper.backward from
    its micro-batch count) is False for the others, whose hooks launch nothing; their bookkeeping is dropped with
    `reset()`, and the syncing pass then all-reduces the accumulated arena bucket by bucket."""

    def __init__(self, arena: FlatArena, process_group=None):
        self.arena, self.group = arena, process_group
        self.world = dist.get_world_size(process_group) if dist.is_initialized() else 1
        self.pending = [0] * len(arena.buckets)
        self.handles = []
        self.launched = [False] * len(arena.buckets)
        self.enabled = True              # tests switch the collective off to take single-rank gradients
        self.sync = True
        if self.world > 1:
            for i, p in enumerate(arena.params):
                p.register_post_accumulate_grad_hook(self._make_hook(arena.bucket_of[i]))
        self.reset()

    def reset(self):
        self.pending = list(self.arena.n_params_in_bucket)
        self.launched = [False] * len(self.arena.buckets)
        self.handles = []
        self.seen = set()

    def _launch(self, b):
        s, e = self.arena.buckets[b]
        if self.arena.grad.is_cuda:
            # NCCL orders the collective after the CURRENT stream only. A bucket can hold gradients written on several
            # streams (3D branch on the main stream, 2D backbone on the side stream): by the time the last hook fires every
            # producing kernel has been enqueued, so waiting on each producer stream here is sufficient.
            cur = torch.cuda.current_stream()
            for st in [torch.cuda.default_stream()] + list(GRAD_STREAMS):
                if st != cur:
                    cur.wait_stream(st)
        self.handles.append(dist.all_reduce(self.arena.grad[s:e], op=dist.ReduceOp.SUM, group=self.group, async_op=True))
        self.launched[b] = True

    def _make_hook(self, b):
        def hook(_p):
            if not (self.enabled and self.sync):
                return
            if id(_p) in self.seen:          # a module used twice in one step fires its (manual) hook twice
                return
            self.seen.add(id(_p))
            self.pending[b] -= 1
            if self.pending[b] == 0 and not self.launched[b]:
                self._launch(b)
        return hook

    def finish(self):
        """Reduce whatever was not launched by hooks (parameters unused this step), then wait."""
        if self.world > 1 and self.enabled:
            for b in range(len(self.arena.buckets)):
                if not self.launched[b]:
                    self._launch(b)
            for h in self.handles:
                h.wait()
        self.reset()


def custom_key(name: str, custom_keys: dict):
    """The `paramwise_cfg.custom_keys` entry that applies to parameter `name`, or None: mmengine's
    DefaultOptimWrapperConstructor takes the longest key contained in the name (equal lengths: alphabetical order)."""
    for k in sorted(sorted(custom_keys), key=len, reverse=True):
        if k in name:
            return custom_keys[k]
    return None


def param_groups(model: nn.Module, lr: float, weight_decay: float, paramwise_cfg: Optional[dict] = None):
    """torch parameter groups laid out as mmengine's DefaultOptimWrapperConstructor lays them out for the same arguments,
    so that group and parameter indices line up with the optimizer state of an mmengine checkpoint: without
    `paramwise_cfg` one group of `model.parameters()`; with it one group per parameter in `named_parameters()` order,
    where a matching `custom_keys` entry sets `lr = lr * lr_mult` and `weight_decay = weight_decay * decay_mult`. Frozen
    parameters get a group of their own without overrides. (Other `paramwise_cfg` keys are not supported.)"""
    if not paramwise_cfg:
        return [{'params': list(model.parameters())}]
    keys = paramwise_cfg.get('custom_keys') or {}
    groups = []
    for name, p in model.named_parameters():
        g = {'params': [p]}
        hit = custom_key(name, keys) if p.requires_grad else None
        if hit is not None:
            g['lr'] = lr * hit.get('lr_mult', 1.)
            g['weight_decay'] = weight_decay * hit.get('decay_mult', 1.)
        groups.append(g)
    return groups


class FusedAdamW(torch.optim.Optimizer):
    """torch.optim.AdamW + global-norm clipping over the arena: two kernel launches per step, no host sync.

    A torch Optimizer with torch AdamW's group keys, so learning-rate schedulers (torch's and mmengine's) attach to it and
    write `group['lr']`, which the next `step()` reads. Every trainable parameter lives in `arena`; parameters outside it
    (frozen) sit in their groups without state. The moments `m`, `v` are arena-shaped; one step count serves all
    parameters. `state_dict()` / `load_state_dict()` speak torch AdamW's format, with two differences: the parameters of a
    group whose lr is 0 keep their moments (torch AdamW would still update them), and a parameter that has no state in a
    loaded dict (torch had never seen its gradient) starts from zero moments under the shared step count."""

    def __init__(self, params, arena: FlatArena, lr=1e-3, betas=(0.9, 0.999), eps=1e-8, weight_decay=1e-4,
                 max_norm=10.0, world_size: int = 1, lr_mult: Optional[torch.Tensor] = None):
        # torch AdamW's defaults (and its checks of the values), so the groups carry exactly its keys
        defaults = torch.optim.AdamW([torch.zeros(1, requires_grad=True)], lr=lr, betas=betas, eps=eps,
                                     weight_decay=weight_decay).defaults
        super().__init__(params, defaults)
        self.arena, self.max_norm, self.world = arena, max_norm, world_size
        self.lr_mult = lr_mult                       # per-element learning-rate multiplier at construction, or None
        self.m = torch.zeros_like(arena.flat)
        self.v = torch.zeros_like(arena.flat)
        self.clip_state = torch.zeros(3, dtype=torch.float32, device=arena.flat.device)   # sumsq, norm, clip coefficient
        self.step_count = 0
        self._offset = {id(p): o for p, o in zip(arena.params, arena.offsets)}
        in_groups = {id(p) for g in self.param_groups for p in g['params']}
        if not self._offset.keys() <= in_groups:
            raise ValueError('FusedAdamW: every arena parameter must be in a parameter group')
        for g in self.param_groups:
            for p in g['params']:
                if p.requires_grad and id(p) not in self._offset:
                    raise ValueError('FusedAdamW: a trainable parameter of the groups has no arena slot')
        # the kernel's group table: the groups that hold arena parameters, in order
        self._slots = [k for k, g in enumerate(self.param_groups) if any(id(p) in self._offset for p in g['params'])]
        self.group_of = None                         # (numel,) uint16 slot of every arena element, several slots only
        if len(self._slots) > 1:
            idx = np.zeros(arena.numel, dtype=np.uint16)
            for s, k in enumerate(self._slots):
                for p in self.param_groups[k]['params']:
                    o = self._offset.get(id(p))
                    if o is not None:
                        idx[o:o + p.numel()] = s
            self.group_of = torch.from_numpy(idx).to(arena.flat.device)

    def step(self, closure=None):
        if closure is not None:
            raise ValueError('FusedAdamW.step takes no closure')
        lr_wd = []
        betas, eps = tuple(self.param_groups[self._slots[0]]['betas']), self.param_groups[self._slots[0]]['eps']
        for k in self._slots:
            g = self.param_groups[k]
            if tuple(g['betas']) != betas or g['eps'] != eps:
                raise ValueError('FusedAdamW: all parameter groups must share betas and eps')
            lr_wd += (float(g['lr']), float(g['weight_decay']))
        lr_wd = torch.tensor(lr_wd, dtype=torch.float32)    # host memory: the kernel launch carries the values
        a = self.arena
        self.step_count += 1
        ws = 1.0 / self.world                         # arena.grad holds the SUM over ranks
        call('esb_grad_clip_coef', ptr(a.grad), a.numel, float(self.max_norm if self.max_norm else 0.), ws,
             ptr(self.clip_state), stream())
        call('esb_adamw_step_groups', ptr(a.flat), ptr(a.grad), ptr(self.m), ptr(self.v), ptr(self.group_of),
             ptr(lr_wd), len(self._slots), a.numel, float(betas[0]), float(betas[1]), float(eps), self.step_count, ws,
             ptr(self.clip_state), stream())

    def zero_grad(self, set_to_none: bool = True):
        """Zero the gradient arena. The parameters' `.grad` stay views of it whatever `set_to_none` says."""
        self.arena.zero_grad()

    def state_dict(self):
        """torch AdamW's format. Parameters are numbered across groups in order; `exp_avg` / `exp_avg_sq` are views of the
        arena's moments (torch's own state_dict also returns its live state tensors)."""
        state, groups, index = {}, [], 0
        for g in self.param_groups:
            packed = {k: v for k, v in g.items() if k != 'params'}
            packed['params'] = list(range(index, index + len(g['params'])))
            index += len(g['params'])
            for i, p in zip(packed['params'], g['params']):
                o = self._offset.get(id(p))
                if o is not None and self.step_count > 0:
                    state[i] = {'step': torch.tensor(float(self.step_count), dtype=torch.float32),
                                'exp_avg': self.m[o:o + p.numel()].view_as(p),
                                'exp_avg_sq': self.v[o:o + p.numel()].view_as(p)}
            groups.append(packed)
        return {'state': state, 'param_groups': groups}

    def load_state_dict(self, state_dict):
        """Load a torch AdamW state dict (written by torch.optim.AdamW, by this class, or by mmengine's
        OptimWrapper.state_dict(), the 'optimizer' entry of a checkpoint) for the same groups: the moments are copied
        into the arena on the current stream, the step count and the groups' lr, initial_lr, weight_decay, betas and eps
        are adopted, and the bf16 shadow is refreshed (a resume loads the model weights, which land in the arena, first).
        Raises ValueError, before changing anything, if the group count, the parameters per group, a moment's shape or
        the steps of the parameters disagree."""
        saved = state_dict['param_groups']
        if len(saved) != len(self.param_groups):
            raise ValueError(f'FusedAdamW.load_state_dict: {len(saved)} parameter groups, expected '
                             f'{len(self.param_groups)}')
        moments, steps = [], set()
        for k, (g, s) in enumerate(zip(self.param_groups, saved)):
            if len(s['params']) != len(g['params']):
                raise ValueError(f'FusedAdamW.load_state_dict: group {k} holds {len(s["params"])} parameters, '
                                 f'expected {len(g["params"])}')
            if s.get('amsgrad') or s.get('maximize'):
                raise ValueError('FusedAdamW.load_state_dict: amsgrad / maximize AdamW states are not supported')
            for p, i in zip(g['params'], s['params']):
                o = self._offset.get(id(p))
                if o is None:
                    continue
                st = state_dict['state'].get(i)
                if st is None:
                    moments.append((p, o, None, None))
                    continue
                for key in ('exp_avg', 'exp_avg_sq'):
                    if tuple(st[key].shape) != tuple(p.shape):
                        raise ValueError(f'FusedAdamW.load_state_dict: {key} of parameter {i} has shape '
                                         f'{tuple(st[key].shape)}, expected {tuple(p.shape)}')
                steps.add(float(st['step']))
                moments.append((p, o, st['exp_avg'], st['exp_avg_sq']))
        if len(steps) > 1:
            raise ValueError(f'FusedAdamW.load_state_dict: the parameters disagree on the step count {sorted(steps)}')
        for p, o, exp_avg, exp_avg_sq in moments:
            n = p.numel()
            if exp_avg is None:
                self.m[o:o + n].zero_()
                self.v[o:o + n].zero_()
            else:
                self.m[o:o + n].copy_(exp_avg.reshape(-1))
                self.v[o:o + n].copy_(exp_avg_sq.reshape(-1))
        self.step_count = int(steps.pop()) if steps else 0
        for g, s in zip(self.param_groups, saved):
            for key in ('lr', 'initial_lr', 'weight_decay', 'betas', 'eps'):
                if key in s:
                    g[key] = s[key]
        self.arena.refresh_bf16()

    @property
    def grad_norm(self):
        return self.clip_state[1]


class OptimWrapper:
    """mmengine's OptimWrapper interface (`update_params(loss)`, `backward`, `step`, `zero_grad`, `param_groups`,
    `get_lr`, `get_momentum`, `state_dict`, `load_state_dict`, and the gradient-accumulation methods `scale_loss`,
    `should_update`, `should_sync`, `optim_context`, `initialize_count_status`) for the arena optimiser `self.optimizer`
    (FusedAdamW), whose groups follow mmengine's `paramwise_cfg` layout. Schedulers attach to `self.optimizer`.

    `accumulative_counts=N` accumulates the gradients of N micro-batches (`update_params` calls) per optimiser step, with
    mmengine's rules: each loss is divided by N (by the remainder `max_counts % N` in a shorter last window), only the
    last micro-batch of a window all-reduces across ranks, and clipping, AdamW, the bf16 shadow refresh and `zero_grad`
    run once per window. The arena adds every micro-batch's gradient to the slots as autograd's `grad += fresh` does.
    The window position is not part of `state_dict()` (as in mmengine)."""

    def __init__(self, model: nn.Module, lr=1e-3, weight_decay=1e-4, max_norm=10.0, process_group=None,
                 bucket_bytes: int = 64 << 20, max_run_ahead: int = 1, paramwise_cfg: Optional[dict] = None,
                 gc_interval: Optional[int] = 200, accumulative_counts: int = 1):
        if not (isinstance(accumulative_counts, int) and accumulative_counts > 0):
            raise ValueError(f'accumulative_counts must be a positive integer, got {accumulative_counts!r}')
        self._accumulative_counts = accumulative_counts
        self._inner_count = 0            # backward passes so far (micro-batches), as mmengine counts them
        self._max_counts = -1            # total training iterations, from initialize_count_status; -1 = unknown
        self._remainder_counts = -1
        # max_run_ahead: how many optimiser steps the host may queue ahead of the device. 1 = while the device finishes step i
        # (tail of backward, all-reduce, clip, AdamW) the host already runs the front of step i+1 (preprocessing, the 2D branch's
        # graph launch, voxelisation) up to its first row-count read: +3.3% on the C2 step (33.3 vs 34.4 ms), 2 adds nothing.
        # (Round 1 kept 0 because unbounded run-ahead "produced" sporadic 100-400 ms stalls; those were the interpreter's
        # garbage collector, see gc_interval below.) 0 = wait for the step's last kernel before returning.
        self.max_run_ahead = max_run_ahead
        self._step_events = []
        # The interpreter's automatic cyclic collector pauses a step for 70-260 ms whenever a generation-1 pass falls into
        # it (4 passes = 4 stalls per 40 steps, none with the collector off; on N ranks the pauses
        # land on different steps of different ranks and every rank waits for the slowest). Like other synchronous
        # data-parallel trainers the wrapper therefore takes the collector over: automatic collection off, one young-generation
        # pass every `gc_interval` optimiser steps, at the same step on every rank, issued while the device is still busy
        # with the step's tail. `gc_interval=None` leaves the interpreter's setting alone.
        self.gc_interval = gc_interval
        self._updates = 0
        if gc_interval:
            import gc
            gc.disable()
        self.arena = FlatArena(model, bucket_bytes)
        world = dist.get_world_size(process_group) if dist.is_initialized() else 1
        self.reducer = DataParallelReducer(self.arena, process_group)
        self.optimizer = FusedAdamW(param_groups(model, lr, weight_decay, paramwise_cfg), self.arena, lr=lr,
                                    weight_decay=weight_decay, max_norm=max_norm, world_size=world,
                                    lr_mult=self._lr_mult(model, paramwise_cfg))
        self.arena.zero_grad()

    def _lr_mult(self, model, paramwise_cfg):
        """mmengine `paramwise_cfg=dict(custom_keys={name_substring: dict(lr_mult=...)})` (the grounding config scales the
        decoder by 0.1 and freezes the text encoder with 0.0: configs/grounding/mv-grounding_8xb12_embodiedscan-vg-9dof.py)
        as ONE per-element multiplier over the arena at construction. The step itself reads each group's lr."""
        keys = (paramwise_cfg or {}).get('custom_keys') or {}
        if not keys:
            return None
        names = {id(p): n for n, p in model.named_parameters()}
        mult = torch.ones(self.arena.numel, dtype=torch.float32, device=self.arena.flat.device)
        for p, o in zip(self.arena.params, self.arena.offsets):
            hit = custom_key(names.get(id(p), ''), keys)
            if hit is not None:
                mult[o:o + p.numel()] = float(hit.get('lr_mult', 1.0))
        return mult

    # what mmengine's hooks and Runner call on an optim wrapper
    @property
    def param_groups(self):
        return self.optimizer.param_groups

    def get_lr(self):
        return {'lr': [g['lr'] for g in self.param_groups]}

    def get_momentum(self):
        return {'momentum': [g['betas'][0] for g in self.param_groups]}

    def state_dict(self):
        return self.optimizer.state_dict()

    def load_state_dict(self, state_dict):
        self.optimizer.load_state_dict(state_dict)

    # ---- gradient accumulation (mmengine OptimWrapper's rules, restated) ------------------------------------------------
    def initialize_count_status(self, model: nn.Module, init_counts: int, max_counts: int):
        """What mmengine's training loops call before the first iteration: `init_counts` iterations done (a resume),
        `max_counts` in all. Sets the micro-batch count and the size of the last, shorter window."""
        import warnings
        self._inner_count = init_counts
        self._max_counts = max_counts
        if self._inner_count % self._accumulative_counts != 0:
            warnings.warn('Resumed iteration number is not divisible by `accumulative_counts`: the gradients of the '
                          'iterations of the interrupted window are lost, which may influence the result slightly.')
        if self._accumulative_counts > 1 and any(isinstance(m, nn.modules.batchnorm._BatchNorm) for m in model.modules()):
            warnings.warn('Gradient accumulation may slightly decrease performance because the model has BatchNorm '
                          'layers (their statistics are those of each micro-batch).')
        self._remainder_counts = self._max_counts % self._accumulative_counts

    def should_update(self) -> bool:
        """True after the last backward pass of a window (or of training): the next step is due."""
        return self._inner_count % self._accumulative_counts == 0 or self._inner_count == self._max_counts

    def should_sync(self) -> bool:
        """True when the next backward pass ends a window: its gradients must be all-reduced across ranks."""
        return ((self._inner_count + 1) % self._accumulative_counts == 0
                or (self._inner_count + 1) == self._max_counts)

    @contextmanager
    def optim_context(self, model: nn.Module):
        """mmengine's context around a micro-batch's forward: a model with `no_sync` (torch DDP) skips the gradient
        synchronisation of a non-syncing micro-batch. The arena's own reducer decides from the count in `backward`, so
        a loop that calls `update_params` without this context is just as correct."""
        if not self.should_sync() and hasattr(model, 'no_sync'):
            with model.no_sync():
                yield
        else:
            yield

    def scale_loss(self, loss: torch.Tensor) -> torch.Tensor:
        """loss / N, or loss / (max_counts % N) in the last, shorter window. N = 1 returns the loss itself."""
        if self._accumulative_counts == 1:
            return loss
        if self._max_counts == -1:
            factor = self._accumulative_counts
        else:
            factor = (self._accumulative_counts if self._inner_count < self._max_counts - self._remainder_counts
                      else self._remainder_counts)
            if factor <= 0:
                raise ValueError('loss factor must be positive: initialize_count_status was called with inconsistent '
                                 f'init_counts={self._inner_count} / max_counts={self._max_counts}')
        return loss / factor

    def backward(self, loss: torch.Tensor):
        """loss.backward(), all-reducing across ranks only if this micro-batch ends a window; counts the micro-batch."""
        sync = self.should_sync()
        self.reducer.sync = sync
        try:
            loss.backward()
        finally:
            self.reducer.sync = True
        if not sync:
            self.reducer.reset()         # the next pass's hooks count their buckets afresh
        self._inner_count += 1

    def step(self):
        """All-reduce what is left, clip + AdamW, refresh the bf16 shadow."""
        self.reducer.finish()
        self.optimizer.step()
        self.arena.refresh_bf16()

    def zero_grad(self):
        self.arena.zero_grad()

    def update_params(self, loss: torch.Tensor):
        """Scale the loss, backward, and once a window is complete: step, zero_grad and the per-step housekeeping."""
        self.backward(self.scale_loss(loss))
        if not self.should_update():
            return
        self.step()
        self.zero_grad()
        self._updates += 1
        if self.gc_interval and self._updates % self.gc_interval == 0:
            import gc
            gc.collect(1)
        if self.arena.flat.is_cuda:
            ev = torch.cuda.Event()
            ev.record()
            self._step_events.append(ev)
            while len(self._step_events) > self.max_run_ahead:
                self._step_events.pop(0).synchronize()


def broadcast_parameters(arena: FlatArena, src: int = 0, process_group=None):
    if dist.is_initialized() and dist.get_world_size(process_group) > 1:
        dist.broadcast(arena.flat, src=src, group=process_group)
    arena.refresh_bf16()
