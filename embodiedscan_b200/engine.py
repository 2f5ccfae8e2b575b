"""Training-step runtime for the hot path: flat parameter/gradient arenas, fused clip + AdamW kernels, and data-parallel
gradient all-reduce over NCCL (NVLink 5 / NVSwitch) launched per bucket as soon as a bucket's gradients are complete.

Replaces, for this path, mmengine's OptimWrapper + MMDistributedDataParallel (†upstream; optimizer and clip settings at
configs/detection/mv-det3d_8xb4_embodiedscan-3d-284class-9dof.py:219-223): one process per GPU, scans sharded across
ranks, the only bulk collective is the gradient SUM (averaged inside the AdamW kernel), no host synchronisation.
"""
from typing import List, Optional

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
            p._esb_uses = 0
            if p.grad is None or p.grad.data_ptr() != self.grad.data_ptr() + 4 * o:
                p.grad = self.grad[o:o + p.numel()].view_as(p)


class DataParallelReducer:
    """Per-bucket asynchronous all-reduce(SUM) of the gradient arena, overlapped with the rest of backward."""

    def __init__(self, arena: FlatArena, process_group=None):
        self.arena, self.group = arena, process_group
        self.world = dist.get_world_size(process_group) if dist.is_initialized() else 1
        self.pending = [0] * len(arena.buckets)
        self.handles = []
        self.launched = [False] * len(arena.buckets)
        self.enabled = True              # tests switch the collective off to take single-rank gradients
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
            if not self.enabled:
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


class FusedAdamW:
    """AdamW + global-norm clipping over the arena: two kernel launches per step, no host sync."""

    def __init__(self, arena: FlatArena, lr=1e-3, betas=(0.9, 0.999), eps=1e-8, weight_decay=1e-4, max_norm=10.0,
                 world_size: int = 1, lr_mult: Optional[torch.Tensor] = None):
        self.arena, self.lr, self.betas, self.eps, self.wd, self.max_norm = arena, lr, betas, eps, weight_decay, max_norm
        self.world = world_size
        self.lr_mult = lr_mult                       # per-element learning-rate multiplier over the arena, or None
        dev = arena.flat.device
        self.m = torch.zeros_like(arena.flat)
        self.v = torch.zeros_like(arena.flat)
        self.state = torch.zeros(3, dtype=torch.float32, device=dev)   # sumsq, norm, clip coefficient
        self.step_count = 0

    def step(self):
        a = self.arena
        self.step_count += 1
        ws = 1.0 / self.world                         # arena.grad holds the SUM over ranks
        call('esb_grad_clip_coef', ptr(a.grad), a.numel, float(self.max_norm if self.max_norm else 0.), ws,
             ptr(self.state), stream())
        call('esb_adamw_step', ptr(a.flat), ptr(a.grad), ptr(self.m), ptr(self.v), ptr(self.lr_mult), a.numel, self.lr, self.betas[0],
             self.betas[1], self.eps, self.wd, self.step_count, ws, ptr(self.state), stream())

    @property
    def grad_norm(self):
        return self.state[1]


class OptimWrapper:
    """``update_params(loss)`` of mmengine's OptimWrapper for the arena optimiser."""

    def __init__(self, model: nn.Module, lr=1e-3, weight_decay=1e-4, max_norm=10.0, process_group=None,
                 bucket_bytes: int = 64 << 20, max_run_ahead: int = 1, paramwise_cfg: Optional[dict] = None,
                 gc_interval: Optional[int] = 200):
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
        self.optimizer = FusedAdamW(self.arena, lr=lr, weight_decay=weight_decay, max_norm=max_norm, world_size=world,
                                    lr_mult=self._lr_mult(model, paramwise_cfg))
        self.arena.zero_grad()

    def _lr_mult(self, model, paramwise_cfg):
        """mmengine `paramwise_cfg=dict(custom_keys={name_substring: dict(lr_mult=...)})` (the grounding config scales the
        decoder by 0.1 and freezes the text encoder with 0.0: configs/grounding/mv-grounding_8xb12_embodiedscan-vg-9dof.py)
        as ONE per-element multiplier over the arena, consumed by the fused AdamW kernel. The longest matching key wins."""
        keys = (paramwise_cfg or {}).get('custom_keys') or {}
        if not keys:
            return None
        names = {id(p): n for n, p in model.named_parameters()}
        mult = torch.ones(self.arena.numel, dtype=torch.float32, device=self.arena.flat.device)
        for p, o in zip(self.arena.params, self.arena.offsets):
            name = names.get(id(p), '')
            hit = [k for k in keys if k in name]
            if hit:
                mult[o:o + p.numel()] = float(keys[max(hit, key=len)].get('lr_mult', 1.0))
        return mult

    def update_params(self, loss: torch.Tensor):
        loss.backward()
        self.reducer.finish()
        self.optimizer.step()
        self.arena.refresh_bf16()
        self.arena.zero_grad()
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
