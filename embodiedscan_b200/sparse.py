"""Sparse-tensor operator surface of the hot path (the subset of the MinkowskiEngine Python API that
``embodiedscan/models/backbones/mink_resnet.py:7-9,58-69`` and
``embodiedscan/models/dense_heads/fcaf3d_head.py:919-984,1101-1145`` touch), backed by ``libesb200.so``.

Semantics (†upstream ME 0.5.x, restated in SURVEY.md Appendix A; frozen by ``oracle/sparse_ref.py``):
  * coordinates int32 ``(N, 4) = [batch, x, y, z]``; duplicates collapse to the FIRST row, first-occurrence order
  * kernel offsets enumerate x fastest: ``k = (dx+1) + 3(dy+1) + 9(dz+1)`` (k3), ``k = dx + 2dy + 4dz`` (k2)
  * stride-2 outputs live at ``floor(c / (2 ts)) * 2 ts``; generative transpose children at ``c + {0,1}^3 * ts/2``,
    child row = ``8 * parent + k``
  * ``A + B`` on different coordinate maps = union (rows of A, then the new rows of B), missing side = 0

Design: a *plan/execute* split. All integer work (dedup, strided maps, kernel maps, pair lists) depends only on the
coordinates, is built once per batch by ``CoordinateManager`` and cached, so every conv of a level shares one map.
"""
import ctypes
import os
from typing import Dict, List, Optional, Tuple

import torch
import torch.nn as nn

from . import _ffi
from ._ffi import call, ptr, query, stream

ACT_NONE, ACT_RELU, ACT_ELU = 0, 1, 2

# bf16 sparse convolutions run on the wgmma tensor-core kernels when the channel counts tile (multiples of 64)
USE_TENSOR_CORES = True
USE_TC_WGRAD = True

# bench.py switches this on to time every sparse-conv launch with CUDA events on the launching stream
CONV_PROFILE = {'enabled': False, 'records': []}


def _timed_conv_call(kind, kmap, cin, cout, dtype, *args):
    if not CONV_PROFILE['enabled']:
        call(*args)
        return
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    call(*args)
    e1.record()
    # keep only the tiny (K+1) pair-offset tensor: holding the KernelMap would pin hundreds of MB of maps per step
    CONV_PROFILE['records'].append((kind, kmap.pairs[2], kmap.K, cin, cout, dtype, e0, e1, kmap.n_in, kmap.n_out))


def _count_use(*params):
    """Forward side of the 'direct' gradient path: a parameter used n times in one step gets its hooks fired after the
    n-th backward contribution (what autograd's AccumulateGrad does for ordinary parameters)."""
    for p in params:
        if p is not None and getattr(p, '_esb_grad_direct', False):
            p._esb_uses = getattr(p, '_esb_uses', 0) + 1


def _fire_grad_hooks(*params):
    for p in params:
        left = getattr(p, '_esb_uses', 1) - 1
        p._esb_uses = max(left, 0)
        if left <= 0:
            for hook in (getattr(p, '_post_accumulate_grad_hooks', None) or {}).values():
                hook(p)       # what autograd's AccumulateGrad would have fired (bucket all-reduce bookkeeping)


def _offsets(kernel_size: int, scale: int) -> List[int]:
    """Kernel offsets (x fastest) in voxel units, multiplied by the input tensor stride."""
    if kernel_size == 1:
        return [0, 0, 0]
    rng = (-1, 0, 1) if kernel_size == 3 else (0, 1)
    out = []
    for dz in rng:
        for dy in rng:
            for dx in rng:
                out += [dx * scale, dy * scale, dz * scale]
    return out


class CoordinateMap:
    """Coordinates of one tensor stride plus their hash table."""

    def __init__(self, coords: torch.Tensor, stride: int, keys=None, vals=None):
        self.coords = coords
        self.stride = stride
        self.n = coords.shape[0]
        self.keys, self.vals = keys, vals
        self._decomp = None

    @property
    def cap(self):
        return self.keys.numel()

    def ensure_table(self):
        if self.keys is None:
            cap = query('esb_hash_capacity', self.n)
            self.keys = torch.empty(cap, dtype=torch.int64, device=self.coords.device)
            self.vals = torch.empty(cap, dtype=torch.int32, device=self.coords.device)
            call('esb_hash_build', ptr(self.coords), self.n, ptr(self.keys), ptr(self.vals), cap, stream())

    def decomposition(self, batch_size: int):
        """(permutations list, seg_off int32 tensor or None if rows are not batch-contiguous)."""
        if self._decomp is None or self._decomp[0] != batch_size:
            b = self.coords[:, 0]
            counts = torch.bincount(b, minlength=batch_size)
            contiguous = bool((b[1:] >= b[:-1]).all().item()) if self.n > 1 else True
            if contiguous:
                off = torch.zeros(batch_size + 1, dtype=torch.int64, device=b.device)
                off[1:] = torch.cumsum(counts, 0)
                off_h = off.tolist()
                ar = torch.arange(self.n, device=b.device)
                perms = [ar[off_h[i]:off_h[i + 1]] for i in range(batch_size)]
                seg_off = off.to(torch.int32)
            else:
                perms = [torch.nonzero(b == i).squeeze(1) for i in range(batch_size)]
                seg_off = None
            self._decomp = (batch_size, perms, seg_off, counts.tolist())
        return self._decomp[1], self._decomp[2], self._decomp[3]


class KernelMap:
    """nbr_out (K, n_out): input row feeding output o through offset k, or -1. Lazy transposed map / pair lists."""

    def __init__(self, nbr_out: torch.Tensor, n_in: int, n_out: int, K: int):
        self.nbr_out, self.n_in, self.n_out, self.K = nbr_out, n_in, n_out, K
        self._nbr_in = None
        self._pairs = None
        self._masks = {}

    @property
    def nbr_in(self):
        if self._nbr_in is None:
            t = torch.empty((self.K, self.n_in), dtype=torch.int32, device=self.nbr_out.device)
            call('esb_kernel_map_transpose', ptr(self.nbr_out), self.K, self.n_out, self.n_in, ptr(t), stream())
            self._nbr_in = t
        return self._nbr_in

    def tile_masks(self, side: str):
        """Per 128-row tile bit mask of used kernel offsets, for nbr_out ('out') or nbr_in ('in')."""
        if side not in self._masks:
            nbr, n = (self.nbr_out, self.n_out) if side == 'out' else (self.nbr_in, self.n_in)
            m = torch.zeros(max((n + 127) // 128, 1), dtype=torch.int32, device=nbr.device)
            call('esb_kmap_tile_masks', ptr(nbr), self.K, n, ptr(m), stream())
            self._masks[side] = m
        return self._masks[side]

    @property
    def pairs(self):
        """(pair_in, pair_out, k_offsets (K+1) device int32, n_pairs upper bound)."""
        if self._pairs is None:
            dev = self.nbr_out.device
            tot = self.K * self.n_out
            pin = torch.empty(max(tot, 1), dtype=torch.int32, device=dev)
            pout = torch.empty(max(tot, 1), dtype=torch.int32, device=dev)
            koff = torch.empty(self.K + 1, dtype=torch.int32, device=dev)
            wsb = query('esb_kmap_pairs_workspace_bytes', self.K, self.n_out)
            ws = torch.empty(wsb, dtype=torch.uint8, device=dev)
            call('esb_kmap_pairs', ptr(self.nbr_out), self.K, self.n_out, ptr(pin), ptr(pout), ptr(koff), ptr(ws), wsb,
                 stream())
            self._pairs = (pin, pout, koff, tot)
        return self._pairs


class CoordinateManager:

    def __init__(self, device):
        self.device = device
        self.maps: Dict[object, CoordinateMap] = {}
        self.kmaps: Dict[object, KernelMap] = {}
        self.in2out: Dict[object, torch.Tensor] = {}
        self.batch_size = 1
        self._uid = 0

    def new_key(self, stride, tag=None):
        self._uid += 1
        return (stride, tag if tag is not None else f'm{self._uid}')

    # ---- construction -------------------------------------------------------------------------------------
    def _unique(self, coords: torch.Tensor, div: int, stride: int):
        n = coords.shape[0]
        cap = query('esb_hash_capacity', n)
        dev = coords.device
        keys = torch.empty(cap, dtype=torch.int64, device=dev)
        vals = torch.empty(cap, dtype=torch.int32, device=dev)
        out = torch.empty((max(n, 1), 4), dtype=torch.int32, device=dev)
        in2out = torch.empty(max(n, 1), dtype=torch.int32, device=dev)
        count = torch.zeros(1, dtype=torch.int32, device=dev)
        wsb = query('esb_coord_unique_workspace_bytes', n)
        ws = torch.empty(wsb, dtype=torch.uint8, device=dev)
        call('esb_coord_unique', ptr(coords), n, div, ptr(keys), ptr(vals), cap, ptr(out), ptr(in2out), ptr(count),
             ptr(ws), wsb, stream())
        c = int(count.item())
        if c < 0:
            raise RuntimeError('esb_coord_unique: coordinate outside the packable range (|xyz| < 32768, batch < 65535)')
        return CoordinateMap(out[:c], stride, keys, vals), in2out[:n]

    def insert(self, coords: torch.Tensor, stride: int = 1, batch_size: Optional[int] = None):
        """Deduplicate raw coordinates. Returns (key, in2out)."""
        cmap, in2out = self._unique(coords.contiguous(), 1, stride)
        key = self.new_key(stride, 'input')
        self.maps[key] = cmap
        if batch_size is None:
            batch_size = int(coords[:, 0].max().item()) + 1 if coords.shape[0] else 1
        self.batch_size = batch_size
        return key, in2out

    def insert_unique(self, coords: torch.Tensor, stride: int):
        key = self.new_key(stride)
        self.maps[key] = CoordinateMap(coords.contiguous(), stride)
        return key

    def stride_key(self, in_key, factor: int = 2):
        ck = ('stride', in_key, factor)
        if ck not in self.kmaps:
            src = self.maps[in_key]
            cmap, in2out = self._unique(src.coords, src.stride * factor, src.stride * factor)
            key = self.new_key(cmap.stride)
            self.maps[key] = cmap
            self.kmaps[ck] = key
            self.in2out[(in_key, key)] = in2out
        return self.kmaps[ck]

    def kernel_map(self, in_key, out_key, kernel_size: int) -> KernelMap:
        ck = ('kmap', in_key, out_key, kernel_size)
        if ck not in self.kmaps:
            src, dst = self.maps[in_key], self.maps[out_key]
            src.ensure_table()
            K = kernel_size ** 3
            offs_arr = _ctypes_int_array(_offsets(kernel_size, src.stride))  # host array, read during the call
            offs = ctypes.cast(offs_arr, ctypes.c_void_p)
            nbr = torch.empty((K, dst.n), dtype=torch.int32, device=self.device)
            call('esb_kernel_map', ptr(dst.coords), dst.n, offs, K, ptr(src.keys), ptr(src.vals), src.cap, ptr(nbr),
                 stream())
            self.kmaps[ck] = KernelMap(nbr, src.n, dst.n, K)
        return self.kmaps[ck]

    def generative_key(self, in_key):
        """Children of a stride-ts map at ts/2; child row = 8*parent + k."""
        ck = ('gen', in_key)
        if ck not in self.kmaps:
            src = self.maps[in_key]
            assert src.stride % 2 == 0, 'generative transpose needs an even tensor stride'
            out = torch.empty((src.n * 8, 4), dtype=torch.int32, device=self.device)
            call('esb_generative_children', ptr(src.coords), src.n, src.stride // 2, ptr(out), stream())
            self.kmaps[ck] = self.insert_unique(out, src.stride // 2)
        return self.kmaps[ck]

    def union_key(self, a_key, b_key):
        """Union of two maps of equal stride: rows of A, then rows of B absent from A (B order).
        Returns (key, map_b) with map_b[j] = union row of B's row j."""
        ck = ('union', a_key, b_key)
        if ck not in self.kmaps:
            A, B = self.maps[a_key], self.maps[b_key]
            assert A.stride == B.stride
            A.ensure_table()
            idx = torch.empty(max(B.n, 1), dtype=torch.int32, device=self.device)[:B.n]
            call('esb_hash_lookup', ptr(B.coords), B.n, ptr(A.keys), ptr(A.vals), A.cap, ptr(idx), stream())
            new = idx < 0
            rank = torch.cumsum(new.to(torch.int32), 0, dtype=torch.int32) - 1 + A.n
            map_b32 = torch.where(new, rank, idx)
            map_b = map_b32.to(torch.int64)
            coords = torch.cat([A.coords, B.coords[new]], 0)
            key = self.insert_unique(coords, A.stride)
            # inverse: union row -> row of B (or -1); the union add is then ONE gather pass, no atomics
            inv_b = torch.full((coords.shape[0], ), -1, dtype=torch.int32, device=self.device)
            inv_b[map_b] = torch.arange(B.n, dtype=torch.int32, device=self.device)
            self.kmaps[ck] = (key, map_b)
            self.kmaps[('union_maps', a_key, b_key)] = (map_b32.contiguous(), inv_b)
        return self.kmaps[ck]


def _ctypes_int_array(vals):
    return (ctypes.c_int * len(vals))(*vals)


# =========================================================================================================
# autograd functions
# =========================================================================================================
class _SparseConv(torch.autograd.Function):

    @staticmethod
    def forward(ctx, x, weight, kmap: KernelMap, cin, cout):
        K = kmap.K
        x = x.contiguous()
        # bf16: the arena's shadow copy when it mirrors the current value (engine.py), else a fresh cast
        w = bf16_operand(weight) if x.dtype == torch.bfloat16 else weight.detach().to(x.dtype).contiguous()
        y = torch.empty((kmap.n_out, cout), dtype=x.dtype, device=x.device)
        tc = USE_TENSOR_CORES and x.dtype == torch.bfloat16 and cin % 64 == 0 and cout % 64 == 0
        if tc:   # the stored (K,cin,cout) kernel is the MN-major B operand: no transpose copy
            _timed_conv_call('fwd', kmap, cin, cout, x.dtype, 'esb_spconv_tc_fwd', ptr(x), ptr(w), ptr(kmap.nbr_out),
                             ptr(kmap.tile_masks('out')), ptr(y), kmap.n_out, cin, cout, K, 1, stream())
        else:
            _timed_conv_call('fwd', kmap, cin, cout, x.dtype, 'esb_spconv_fwd', ptr(x), ptr(w), ptr(kmap.nbr_out),
                             ptr(y), kmap.n_out, cin, cout, K, 0, 0, _ffi.dtype_code(x.dtype), stream())
        ctx.save_for_backward(x, w)
        ctx.kmap, ctx.cin, ctx.cout, ctx.wshape, ctx.tc, ctx.weight = kmap, cin, cout, weight.shape, tc, weight
        if ctx.needs_input_grad[1]:
            _count_use(weight)
        return y

    @staticmethod
    def backward(ctx, dy):
        x, w = ctx.saved_tensors
        kmap, cin, cout = ctx.kmap, ctx.cin, ctx.cout
        dy = dy.contiguous()
        code = _ffi.dtype_code(x.dtype)
        dx = dw = None
        if ctx.needs_input_grad[0]:
            dx = torch.empty((kmap.n_in, cin), dtype=x.dtype, device=x.device)
            # dgrad = the forward kernel on the input-stationary map with W read transposed
            if ctx.tc:   # (K,cin,cout) already is the K-major B operand of the transposed problem
                _timed_conv_call('dgrad', kmap, cout, cin, x.dtype, 'esb_spconv_tc_fwd', ptr(dy), ptr(w), ptr(kmap.nbr_in),
                                 ptr(kmap.tile_masks('in')), ptr(dx), kmap.n_in, cout, cin, kmap.K, 0, stream())
            else:
                _timed_conv_call('dgrad', kmap, cout, cin, x.dtype, 'esb_spconv_fwd', ptr(dy), ptr(w), ptr(kmap.nbr_in),
                                 ptr(dx), kmap.n_in, cout, cin, kmap.K, 1, 0, code, stream())
        if ctx.needs_input_grad[1]:
            pin, pout, koff, tot = kmap.pairs
            weight = ctx.weight
            direct = getattr(weight, '_esb_grad_direct', False) and weight.grad is not None
            # arena parameters: the kernel accumulates straight into the flat gradient buffer (no zeros + add_ pass)
            dw = weight.grad if direct else torch.zeros((kmap.K, cin, cout), dtype=torch.float32, device=x.device)
            if ctx.tc and USE_TC_WGRAD:
                _timed_conv_call('wgrad', kmap, cin, cout, x.dtype, 'esb_spconv_tc_wgrad', ptr(x), ptr(dy), ptr(pin),
                                 ptr(pout), ptr(koff), ptr(dw), tot, cin, cout, kmap.K, stream())
            else:
                _timed_conv_call('wgrad', kmap, cin, cout, x.dtype, 'esb_spconv_wgrad', ptr(x), ptr(dy), ptr(pin),
                                 ptr(pout), ptr(koff), ptr(dw), tot, cin, cout, kmap.K, code, stream())
            if direct:
                _fire_grad_hooks(weight)
                dw = None
            else:
                dw = dw.view(ctx.wshape)
        return dx, dw, None, None, None


class _ShadowCast(torch.autograd.Function):
    """fp32 parameter -> its bf16 operand copy (the arena's shadow when it is fresh, else a cast), connected to autograd."""

    @staticmethod
    def forward(ctx, p):
        return bf16_operand(p)

    @staticmethod
    def backward(ctx, g):
        return g.float()


def bf16_operand(p: torch.Tensor) -> torch.Tensor:
    """The bf16 copy of a parameter that kernels read: the arena shadow if it mirrors the CURRENT value (engine.FlatArena
    stamps the parameter version at every refresh; load_state_dict / init / manual edits bump it), else a fresh cast."""
    sh = getattr(p, '_esb_bf16', None)
    if sh is not None and getattr(p, '_esb_bf16_version', None) == p._version:
        return sh
    return p.detach().to(torch.bfloat16).contiguous()


_IDENTITY_MAPS = {}


def _identity_map(n: int, device):
    """Kernel map of a dense rows GEMM: ONE offset whose neighbour of row i is row i (cached per row count)."""
    key = (n, str(device))
    m = _IDENTITY_MAPS.get(key)
    if m is None:
        if len(_IDENTITY_MAPS) > 64:
            _IDENTITY_MAPS.clear()
        ar = torch.arange(n, dtype=torch.int32, device=device)
        masks = torch.ones(max((n + 127) // 128, 1), dtype=torch.int32, device=device)
        koff = torch.tensor([0, n], dtype=torch.int32, device=device)
        m = _IDENTITY_MAPS[key] = (ar, masks, koff)
    return m


class _RowsGemmTC(torch.autograd.Function):
    """y (N, cout) = x (N, cin) @ w (cin, cout) in bf16 on the sparse-conv tensor-core kernels with the identity map:
    forward = spconv_tc_fwd (w as the MN-major B operand), dx = the same kernel with w read K-major, dw = spconv_tc_wgrad
    over the identity pair list. The dense contractions of the head (generative transpose, 1x1 convolutions;
    embodiedscan/models/dense_heads/fcaf3d_head.py:937-941,970-982) stay on the library's own kernels."""

    @staticmethod
    def forward(ctx, x, w):
        x = x.contiguous()
        w = w.contiguous()
        N, cin = x.shape
        cout = w.shape[1]
        y = torch.empty((N, cout), dtype=torch.bfloat16, device=x.device)
        ar, masks, koff = _identity_map(N, x.device)
        if N:
            call('esb_spconv_tc_fwd', ptr(x), ptr(w), ptr(ar), ptr(masks), ptr(y), N, cin, cout, 1, 1, stream())
        ctx.save_for_backward(x, w)
        return y

    @staticmethod
    def backward(ctx, dy):
        x, w = ctx.saved_tensors
        N, cin = x.shape
        cout = w.shape[1]
        dy = dy.contiguous()
        ar, masks, koff = _identity_map(N, x.device)
        dx = dw = None
        if ctx.needs_input_grad[0]:
            dx = torch.empty_like(x)
            if N:
                call('esb_spconv_tc_fwd', ptr(dy), ptr(w), ptr(ar), ptr(masks), ptr(dx), N, cout, cin, 1, 0, stream())
        if ctx.needs_input_grad[1]:
            dw = torch.zeros((cin, cout), dtype=torch.float32, device=x.device)
            if N:
                call('esb_spconv_tc_wgrad', ptr(x), ptr(dy), ptr(ar), ptr(ar), ptr(koff), ptr(dw), N, cin, cout, 1, stream())
        return dx, dw


def rows_gemm(x: torch.Tensor, w: torch.Tensor) -> torch.Tensor:
    """x (N, cin) @ w (cin, cout). bf16 CUDA rows with channel counts that tile (multiples of 64) run on the library's
    tensor-core kernels; anything else (fp32 parity arithmetic, odd widths) is a plain matmul."""
    if (USE_TENSOR_CORES and x.is_cuda and x.dtype == torch.bfloat16 and w.dtype == torch.bfloat16 and x.shape[1] % 64 == 0
            and w.shape[1] % 64 == 0):
        return _RowsGemmTC.apply(x, w)
    return x @ w.to(x.dtype)


def weight_operand(p: torch.Tensor, dtype) -> torch.Tensor:
    """A parameter as the operand of compute dtype `dtype`, connected to autograd."""
    if dtype == torch.bfloat16 and p.is_cuda and p.dtype == torch.float32:
        return _ShadowCast.apply(p)
    return p.to(dtype)


class _UnionAdd(torch.autograd.Function):
    """out = A (rows 0..nA of the union) + B scattered by map_b, as one row-gather pass (csrc/spops.cu::gather2_rows_kernel);
    backward: dA = the first nA rows of dOut, dB = dOut gathered by map_b."""

    @staticmethod
    def forward(ctx, fa, fb, map_b32, inv_b, n_union):
        fa, fb = fa.contiguous(), fb.contiguous()
        out = torch.empty((n_union, fa.shape[1]), dtype=fa.dtype, device=fa.device)
        call('esb_gather2_rows', ptr(fa), None, fa.shape[0], ptr(fb), ptr(inv_b), ptr(out), n_union, fa.shape[1],
             _ffi.dtype_code(fa.dtype), stream())
        ctx.save_for_backward(map_b32)
        ctx.na = fa.shape[0]
        return out

    @staticmethod
    def backward(ctx, dout):
        (map_b32, ) = ctx.saved_tensors
        dout = dout.contiguous()
        da = dout[:ctx.na] if ctx.needs_input_grad[0] else None
        db = None
        if ctx.needs_input_grad[1]:
            db = torch.empty((map_b32.shape[0], dout.shape[1]), dtype=dout.dtype, device=dout.device)
            call('esb_gather2_rows', ptr(dout), ptr(map_b32), dout.shape[0], None, None, ptr(db), map_b32.shape[0],
                 dout.shape[1], _ffi.dtype_code(dout.dtype), stream())
        return da, db, None, None, None


class _MaxPool(torch.autograd.Function):

    @staticmethod
    def forward(ctx, x, kmap: KernelMap):
        x = x.contiguous()
        C = x.shape[1]
        y = torch.empty((kmap.n_out, C), dtype=x.dtype, device=x.device)
        arg = torch.empty((kmap.n_out, C), dtype=torch.int32, device=x.device)
        call('esb_maxpool_fwd', ptr(x), ptr(kmap.nbr_out), ptr(y), ptr(arg), kmap.n_out, C, kmap.K,
             _ffi.dtype_code(x.dtype), stream())
        ctx.save_for_backward(arg)
        ctx.n_in, ctx.n_out = kmap.n_in, kmap.n_out
        return y

    @staticmethod
    def backward(ctx, dy):
        (arg, ) = ctx.saved_tensors
        dy = dy.contiguous()
        dx = torch.zeros((ctx.n_in, dy.shape[1]), dtype=dy.dtype, device=dy.device)
        call('esb_maxpool_bwd', ptr(dy), ptr(arg), ptr(dx), ctx.n_out, dy.shape[1], _ffi.dtype_code(dy.dtype), stream())
        return dx, None


class _SegNorm(torch.autograd.Function):
    """y = act(norm(x) * gamma + beta + res) with batch statistics per segment (BatchNorm: one segment)."""

    @staticmethod
    def forward(ctx, x, res, gamma, beta, seg_off, row_seg, S, max_rows, eps, running_mean, running_var, momentum, act):
        x = x.contiguous()
        N, C = x.shape
        dev = x.device
        y = torch.empty_like(x)
        g = gamma.detach() if gamma is not None else None      # fp32 contiguous parameters: used as is
        b = beta.detach() if beta is not None else None
        assert (g is None or (g.dtype == torch.float32 and g.is_contiguous())) and \
            (b is None or (b.dtype == torch.float32 and b.is_contiguous()))
        resc = res.contiguous() if res is not None else None
        if S == 1 and x.dtype == torch.bfloat16 and C % 8 == 0 and 8 <= C <= 2048 and N > 0:
            # BatchNorm on the throughput path: one shifted single-pass statistics kernel + one apply kernel
            stats = torch.empty((4, C), dtype=torch.float32, device=dev)
            call('esb_batchnorm_fwd_fused', ptr(x), ptr(resc), N, C, ptr(g), ptr(b), eps, ptr(running_mean), ptr(running_var),
                 momentum, act, ptr(stats), ptr(y), _ffi.dtype_code(x.dtype), stream())
            mean, rstd = stats[2:3], stats[3:4]
        else:
            mean = torch.empty((S, C), dtype=torch.float32, device=dev)
            rstd = torch.empty((S, C), dtype=torch.float32, device=dev)
            call('esb_norm_fwd', ptr(x), ptr(resc), ptr(seg_off), ptr(row_seg), S, N, max_rows, C, ptr(g), ptr(b), eps,
                 ptr(running_mean), ptr(running_var), momentum, act, ptr(mean), ptr(rstd), ptr(y), _ffi.dtype_code(x.dtype),
                 stream())
        ctx.save_for_backward(x, y, mean, rstd, g, seg_off, row_seg)   # None entries are allowed
        ctx.meta = (S, max_rows, act, res is not None, gamma.shape if gamma is not None else None,
                    beta.shape if beta is not None else None)
        ctx.params = (gamma, beta)
        if S == 1 and gamma is not None and beta is not None and ctx.needs_input_grad[2]:
            _count_use(gamma, beta)
        return y

    @staticmethod
    def backward(ctx, dy):
        x, y, mean, rstd, g, seg_off, row_seg = ctx.saved_tensors
        S, max_rows, act, has_res, gshape, bshape = ctx.meta
        N, C = x.shape
        dy = dy.contiguous()
        gamma, beta = ctx.params
        direct = (S == 1 and gamma is not None and beta is not None and getattr(gamma, '_esb_grad_direct', False)
                  and getattr(beta, '_esb_grad_direct', False) and gamma.grad is not None and beta.grad is not None)
        if direct:   # the column sums ARE d(beta), d(gamma): accumulate them in the arena's (zeroed) gradient slots
            sg, sgx = beta.grad, gamma.grad
        else:
            sg = torch.empty((S, C), dtype=torch.float32, device=x.device)
            sgx = torch.empty((S, C), dtype=torch.float32, device=x.device)
        dx = torch.empty_like(x)
        dres = torch.empty_like(x) if has_res else None
        call('esb_norm_bwd', ptr(x), ptr(y), ptr(dy), ptr(seg_off), ptr(row_seg), S, N, max_rows, C, ptr(mean), ptr(rstd),
             ptr(g), act, ptr(sg), ptr(sgx), ptr(dx), ptr(dres), 0 if direct else 1, _ffi.dtype_code(x.dtype), stream())
        if direct:
            _fire_grad_hooks(gamma, beta)
            return dx, dres, None, None, None, None, None, None, None, None, None, None, None
        if S == 1:       # BatchNorm: the (1,C) sums ARE the parameter gradients (no reduction kernel)
            dgamma = sgx.view(gshape) if gshape is not None else None
            dbeta = sg.view(bshape) if bshape is not None else None
        else:
            dgamma = sgx.sum(0).view(gshape) if gshape is not None else None
            dbeta = sg.sum(0).view(bshape) if bshape is not None else None
        return dx, dres, dgamma, dbeta, None, None, None, None, None, None, None, None, None


def seg_norm(x, gamma, beta, seg_off, row_seg, S, max_rows, eps, act=ACT_NONE, res=None, running_mean=None,
             running_var=None, momentum=0.1):
    return _SegNorm.apply(x, res, gamma, beta, seg_off, row_seg, S, max_rows, eps, running_mean, running_var, momentum,
                          act)


def norm_apply_eval(x, mean, var, gamma, beta, eps, act=ACT_NONE, res=None):
    """Inference-mode BatchNorm (+res, +act) with running statistics; no autograd."""
    x = x.contiguous()
    N, C = x.shape
    m = mean.float().contiguous().view(1, C)
    rstd = torch.rsqrt(var.float() + eps).contiguous().view(1, C)
    y = torch.empty_like(x)
    resc = res.contiguous() if res is not None else None
    call('esb_norm_apply', ptr(x), ptr(resc), None, N, C, ptr(m), ptr(rstd), ptr(gamma.detach().float().contiguous()),
         ptr(beta.detach().float().contiguous()), act, ptr(y), _ffi.dtype_code(x.dtype), stream())
    return y


# =========================================================================================================
# SparseTensor + modules (ME-named so reference-style model code reads the same)
# =========================================================================================================
def _spread3(v: torch.Tensor) -> torch.Tensor:
    """Bits of a 16-bit value moved to every third position (int64), the classic Morton "part1by2"."""
    v = v & 0xffff
    v = (v | (v << 32)) & 0x1f00000000ffff
    v = (v | (v << 16)) & 0x1f0000ff0000ff
    v = (v | (v << 8)) & 0x100f00f00f00f00f
    v = (v | (v << 4)) & 0x10c30c30c30c30c3
    v = (v | (v << 2)) & 0x1249249249249249
    return v


def morton_order(coords: torch.Tensor) -> torch.Tensor:
    """Stable permutation that sorts raw voxel coordinates (N,4) [b,x,y,z] by (scan, Z-order curve of xyz).
    Z-order is hierarchical: the first-occurrence parents of sorted rows (stride-2 maps), the children ``8*parent+k``
    of generative maps and the appended rows of unions all inherit spatial locality from this one sort, so a 128-row
    conv tile gathers from a compact neighbourhood. Stable => points of one voxel keep their input order, i.e. the
    first-occurrence dedup picks the same point (and feature) as without the sort; only the ROW ORDER changes."""
    c = coords.to(torch.int64)
    key = (c[:, 0] << 48) | _spread3(c[:, 1] + 32768) | (_spread3(c[:, 2] + 32768) << 1) | (_spread3(c[:, 3] + 32768) << 2)
    return torch.sort(key, stable=True).indices


def row_order() -> str:
    """'input' (default: rows in first-occurrence order of the input points, the order the parity tests pin) or
    'morton' (opt-in through ESB200_ROW_ORDER=morton; same voxels, same features, Z-ordered rows)."""
    return os.environ.get('ESB200_ROW_ORDER', 'input')


class SparseTensor:

    def __init__(self, features: torch.Tensor, coordinates: Optional[torch.Tensor] = None, coordinate_map_key=None,
                 coordinate_manager: Optional[CoordinateManager] = None, batch_size: Optional[int] = None):
        if coordinates is not None:
            assert coordinate_map_key is None
            if coordinate_manager is None:
                coordinate_manager = CoordinateManager(features.device)
            coords = coordinates.to(device=features.device, dtype=torch.int32)
            if row_order() == 'morton' and coords.shape[0]:
                order = morton_order(coords)
                coords, features = coords[order].contiguous(), features[order]
            key, in2out = coordinate_manager.insert(coords, 1, batch_size)
            n = coordinate_manager.maps[key].n
            # first occurrence wins: scatter in reverse order so the lowest row index is written last
            first = torch.full((n, ), coords.shape[0], dtype=torch.int64, device=features.device)
            first.scatter_reduce_(0, in2out.to(torch.int64), torch.arange(coords.shape[0], device=features.device),
                                  reduce='amin', include_self=True)
            features = features[first]
            coordinate_map_key = key
        self.F = features
        self.coordinate_map_key = coordinate_map_key
        self.coordinate_manager = coordinate_manager

    # ME attribute names
    @property
    def features(self):
        return self.F

    @property
    def cmap(self) -> CoordinateMap:
        return self.coordinate_manager.maps[self.coordinate_map_key]

    @property
    def C(self):
        return self.cmap.coords

    @property
    def coordinates(self):
        return self.cmap.coords

    @property
    def tensor_stride(self):
        s = self.cmap.stride
        return [s, s, s]

    @property
    def device(self):
        return self.F.device

    def __len__(self):
        return self.F.shape[0]

    @property
    def decomposition_permutations(self):
        return self.cmap.decomposition(self.coordinate_manager.batch_size)[0]

    @property
    def decomposed_coordinates(self):
        perms = self.decomposition_permutations
        c = self.cmap.coords
        return [c[p, 1:] for p in perms]

    @property
    def decomposed_features(self):
        return [self.F[p] for p in self.decomposition_permutations]

    def replace_feature(self, f):
        return SparseTensor(f, coordinate_map_key=self.coordinate_map_key, coordinate_manager=self.coordinate_manager)

    def __add__(self, other: 'SparseTensor') -> 'SparseTensor':
        mgr = self.coordinate_manager
        if other.coordinate_map_key == self.coordinate_map_key:
            return self.replace_feature(self.F + other.F)
        key, map_b = mgr.union_key(self.coordinate_map_key, other.coordinate_map_key)
        n = mgr.maps[key].n
        if self.F.is_cuda and self.F.shape[1] % 8 == 0 and self.F.dtype in (torch.float32, torch.bfloat16):
            map_b32, inv_b = mgr.kmaps[('union_maps', self.coordinate_map_key, other.coordinate_map_key)]
            out = _UnionAdd.apply(self.F, other.F.to(self.F.dtype), map_b32, inv_b, n)
        else:
            pad = torch.zeros((n - self.F.shape[0], self.F.shape[1]), dtype=self.F.dtype, device=self.F.device)
            out = torch.cat([self.F, pad], 0).index_add(0, map_b, other.F.to(self.F.dtype))
        return SparseTensor(out, coordinate_map_key=key, coordinate_manager=mgr)

    def features_at_coordinates(self, query: torch.Tensor) -> torch.Tensor:
        """Multilinear interpolation of the features at continuous coordinates [b, x, y, z] on this tensor's lattice
        (absent lattice points contribute 0). †upstream ME `features_at_coordinates`; used by FCAF3D `_prune`."""
        cm = self.cmap
        cm.ensure_table()
        ts = cm.stride
        if (query.is_cuda and self.F.dtype in (torch.float32, torch.bfloat16) and ts & (ts - 1) == 0
                and (not query.is_floating_point() or bool(getattr(query, '_esb_integer', False)))):
            qi = query.to(torch.int32).contiguous()            # integer lattice queries (child coordinates): one kernel
            out = torch.empty((qi.shape[0], self.F.shape[1]), dtype=torch.float32, device=qi.device)
            call('esb_interp_features', ptr(qi), qi.shape[0], ptr(cm.keys), ptr(cm.vals), cm.cap, ptr(self.F.contiguous()),
                 self.F.shape[1], ts, _ffi.dtype_code(self.F.dtype), ptr(out), stream())
            return out
        q = query.float()
        b = q[:, 0].to(torch.int32)
        base = torch.floor(q[:, 1:] / ts)
        frac = q[:, 1:] / ts - base
        base = base.to(torch.int32) * ts
        out = torch.zeros((q.shape[0], self.F.shape[1]), dtype=torch.float32, device=q.device)
        idx = torch.empty(q.shape[0], dtype=torch.int32, device=q.device)
        for k in range(8):
            d = torch.tensor([k & 1, (k >> 1) & 1, (k >> 2) & 1], device=q.device)
            w = torch.where(d.bool(), frac, 1 - frac).prod(1)
            c = torch.cat([b[:, None], base + (d * ts).to(torch.int32)], 1).contiguous()
            call('esb_hash_lookup', ptr(c), c.shape[0], ptr(cm.keys), ptr(cm.vals), cm.cap, ptr(idx), stream())
            hit = idx >= 0
            out += torch.where(hit[:, None], self.F.float()[idx.clamp(min=0).long()] * w[:, None], 0.)
        return out

    def dense(self, shape, min_coordinate=None):
        """Scatter to a dense (B, C, X, Y, Z) tensor on the tensor-stride lattice (ME `.dense`)."""
        cm = self.cmap
        ts = cm.stride
        c = cm.coords.long()
        mn = torch.zeros(3, dtype=torch.long, device=c.device) if min_coordinate is None else \
            torch.as_tensor(min_coordinate, device=c.device).long().view(-1)[-3:]
        ijk = (c[:, 1:] - mn) // ts
        B, Cc, X, Y, Z = shape
        ok = ((ijk >= 0) & (ijk < torch.tensor([X, Y, Z], device=c.device))).all(1)
        out = torch.zeros((B, X, Y, Z, Cc), dtype=self.F.dtype, device=self.F.device)
        out[c[ok, 0], ijk[ok, 0], ijk[ok, 1], ijk[ok, 2]] = self.F[ok]
        return out.permute(0, 4, 1, 2, 3), mn, ts


def batched_coordinates(coords_list, device=None):
    """ME.utils.batched_coordinates: floor float coordinates, prepend the batch index."""
    out = []
    for b, c in enumerate(coords_list):
        c = torch.floor(c).to(torch.int32) if c.is_floating_point() else c.to(torch.int32)
        out.append(torch.cat([torch.full((c.shape[0], 1), b, dtype=torch.int32, device=c.device), c], 1))
    res = torch.cat(out, 0)
    return res.to(device) if device is not None else res


def batch_sparse_collate(data, device=None):
    """ME.utils.batch_sparse_collate for [(coords, feats), ...]."""
    coords = batched_coordinates([d[0] for d in data], device=device)
    feats = torch.cat([d[1] for d in data], 0)
    return coords, (feats.to(device) if device is not None else feats)


def cat(a: SparseTensor, b: SparseTensor) -> SparseTensor:
    assert a.coordinate_map_key == b.coordinate_map_key, 'ME.cat requires the same coordinate map'
    return a.replace_feature(torch.cat([a.F, b.F.to(a.F.dtype)], 1))


def kaiming_normal_(tensor, mode='fan_out', nonlinearity='relu'):
    """ME.utils.kaiming_normal_ for kernels shaped (K, Cin, Cout) or (Cin, Cout)."""
    if tensor.dim() == 3:
        K, cin, cout = tensor.shape
    else:
        K, (cin, cout) = 1, tensor.shape
    fan = cout * K if mode == 'fan_out' else cin * K
    gain = nn.init.calculate_gain(nonlinearity)
    std = gain / fan ** 0.5
    with torch.no_grad():
        return tensor.normal_(0, std)


class MinkowskiConvolution(nn.Module):

    def __init__(self, in_channels, out_channels, kernel_size=1, stride=1, bias=False, dimension=3):
        super().__init__()
        assert dimension == 3 and kernel_size in (1, 2, 3) and stride in (1, 2)
        self.in_channels, self.out_channels, self.kernel_size, self.stride = in_channels, out_channels, kernel_size, stride
        K = kernel_size ** 3
        shape = (in_channels, out_channels) if K == 1 else (K, in_channels, out_channels)
        self.kernel = nn.Parameter(torch.empty(shape))
        self.bias = nn.Parameter(torch.zeros(1, out_channels)) if bias else None
        # ME default init: uniform(-stdv, stdv), stdv = 1/sqrt(in_channels * K)
        stdv = 1.0 / (in_channels * K) ** 0.5
        with torch.no_grad():
            self.kernel.uniform_(-stdv, stdv)
            if self.bias is not None:
                self.bias.uniform_(-stdv, stdv)

    def forward(self, x: SparseTensor) -> SparseTensor:
        mgr = x.coordinate_manager
        in_key = x.coordinate_map_key
        if self.kernel_size == 1 and self.stride == 1:
            y = rows_gemm(x.F, weight_operand(self.kernel, x.F.dtype))   # dense GEMM over rows, identity kernel map
            out_key = in_key
        else:
            out_key = mgr.stride_key(in_key, self.stride) if self.stride > 1 else in_key
            kmap = mgr.kernel_map(in_key, out_key, self.kernel_size)
            y = _SparseConv.apply(x.F, self.kernel, kmap, self.in_channels, self.out_channels)
        if self.bias is not None:
            y = y + self.bias.to(y.dtype)
        return SparseTensor(y, coordinate_map_key=out_key, coordinate_manager=mgr)


class MinkowskiGenerativeConvolutionTranspose(nn.Module):
    """k2 s2 generative transpose conv: a dense GEMM (N_in, Cin) x (Cin, 8*Cout); child row = 8*parent + k."""

    def __init__(self, in_channels, out_channels, kernel_size=2, stride=2, bias=False, dimension=3):
        super().__init__()
        assert kernel_size == 2 and stride == 2 and dimension == 3 and not bias
        self.in_channels, self.out_channels = in_channels, out_channels
        self.kernel = nn.Parameter(torch.empty(8, in_channels, out_channels))
        stdv = 1.0 / (in_channels * 8) ** 0.5
        with torch.no_grad():
            self.kernel.uniform_(-stdv, stdv)

    def forward(self, x: SparseTensor) -> SparseTensor:
        mgr = x.coordinate_manager
        out_key = mgr.generative_key(x.coordinate_map_key)
        w = weight_operand(self.kernel, x.F.dtype).permute(1, 0, 2).reshape(self.in_channels, 8 * self.out_channels)
        y = rows_gemm(x.F, w).view(-1, self.out_channels)
        return SparseTensor(y, coordinate_map_key=out_key, coordinate_manager=mgr)


class MinkowskiBatchNorm(nn.Module):

    def __init__(self, num_features, eps=1e-5, momentum=0.1):
        super().__init__()
        self.bn = nn.BatchNorm1d(num_features, eps=eps, momentum=momentum)

    def forward(self, x: SparseTensor, act=ACT_NONE, res=None) -> SparseTensor:
        return x.replace_feature(batch_norm_rows(x.F, self.bn, self.training, act, res))


def batch_norm_rows(f, bn: nn.BatchNorm1d, training: bool, act=ACT_NONE, res=None):
    if training:
        N = f.shape[0]
        # (num_batches_tracked is only read when momentum is None; it is advanced once per step by the optimiser wrapper)
        return seg_norm(f, bn.weight, bn.bias, None, None, 1, N, bn.eps, act, res, bn.running_mean, bn.running_var,
                        bn.momentum)
    return norm_apply_eval(f, bn.running_mean, bn.running_var, bn.weight, bn.bias, bn.eps, act, res)


class MinkowskiInstanceNorm(nn.Module):
    """Per (scan, channel) normalisation over that scan's rows, eps 1e-8 (†upstream ME), affine (1, C)."""

    def __init__(self, num_features):
        super().__init__()
        self.num_features = num_features
        self.eps = 1e-8
        self.weight = nn.Parameter(torch.ones(1, num_features))
        self.bias = nn.Parameter(torch.zeros(1, num_features))

    def forward(self, x: SparseTensor, act=ACT_NONE) -> SparseTensor:
        B = x.coordinate_manager.batch_size
        perms, seg_off, counts = x.cmap.decomposition(B)
        assert seg_off is not None, 'InstanceNorm expects batch-contiguous rows'
        row_seg = x.cmap.coords[:, 0].contiguous()
        y = seg_norm(x.F, self.weight, self.bias, seg_off, row_seg, B, max(counts) if counts else 0, self.eps, act)
        return x.replace_feature(y)


class _Act(nn.Module):
    code = ACT_NONE

    def __init__(self, inplace=False):
        super().__init__()

    def forward(self, x: SparseTensor) -> SparseTensor:
        f = torch.relu(x.F) if self.code == ACT_RELU else torch.nn.functional.elu(x.F)
        return x.replace_feature(f)


class MinkowskiReLU(_Act):
    code = ACT_RELU


class MinkowskiELU(_Act):
    code = ACT_ELU


class MinkowskiMaxPooling(nn.Module):

    def __init__(self, kernel_size=2, stride=2, dimension=3):
        super().__init__()
        assert kernel_size == 2 and stride == 2 and dimension == 3
        self.kernel_size, self.stride = kernel_size, stride

    def forward(self, x: SparseTensor) -> SparseTensor:
        mgr = x.coordinate_manager
        out_key = mgr.stride_key(x.coordinate_map_key, self.stride)
        kmap = mgr.kernel_map(x.coordinate_map_key, out_key, self.kernel_size)
        return SparseTensor(_MaxPool.apply(x.F, kmap), coordinate_map_key=out_key, coordinate_manager=mgr)


class MinkowskiPruning(nn.Module):

    def forward(self, x: SparseTensor, mask: torch.Tensor) -> SparseTensor:
        if bool(mask.all().item()):
            return x
        mgr = x.coordinate_manager
        key = mgr.insert_unique(x.cmap.coords[mask], x.cmap.stride)
        return SparseTensor(x.F[mask], coordinate_map_key=key, coordinate_manager=mgr)


def conv_norm_act(conv, norm, act_code, x: SparseTensor, res=None, training=True) -> SparseTensor:
    """conv -> BatchNorm(+res)(+act) with the normalisation, residual add and activation fused in one kernel."""
    y = conv(x)
    return y.replace_feature(batch_norm_rows(y.F, norm.bn, training, act_code, res))


class BasicBlock(nn.Module):
    """ME.modules.resnet_block.BasicBlock: conv3-BN-ReLU-conv3-BN-(+downsample(x))-ReLU."""
    expansion = 1

    def __init__(self, inplanes, planes, stride=1, dilation=1, downsample=None, bn_momentum=0.1, dimension=3):
        super().__init__()
        self.conv1 = MinkowskiConvolution(inplanes, planes, kernel_size=3, stride=stride, dimension=dimension)
        self.norm1 = MinkowskiBatchNorm(planes, momentum=bn_momentum)
        self.conv2 = MinkowskiConvolution(planes, planes, kernel_size=3, stride=1, dimension=dimension)
        self.norm2 = MinkowskiBatchNorm(planes, momentum=bn_momentum)
        self.relu = MinkowskiReLU(inplace=True)
        self.downsample = downsample

    def forward(self, x: SparseTensor) -> SparseTensor:
        out = conv_norm_act(self.conv1, self.norm1, ACT_RELU, x, training=self.training)
        if self.downsample is not None:
            r = self.downsample[0](x)
            residual = batch_norm_rows(r.F, self.downsample[1].bn, self.training)
        else:
            residual = x.F
        return conv_norm_act(self.conv2, self.norm2, ACT_RELU, out, res=residual, training=self.training)


class Bottleneck(nn.Module):
    """ME.modules.resnet_block.Bottleneck: 1x1-BN-ReLU, 3x3(stride)-BN-ReLU, 1x1(x4)-BN, +res, ReLU."""
    expansion = 4

    def __init__(self, inplanes, planes, stride=1, dilation=1, downsample=None, bn_momentum=0.1, dimension=3):
        super().__init__()
        self.conv1 = MinkowskiConvolution(inplanes, planes, kernel_size=1, dimension=dimension)
        self.norm1 = MinkowskiBatchNorm(planes, momentum=bn_momentum)
        self.conv2 = MinkowskiConvolution(planes, planes, kernel_size=3, stride=stride, dimension=dimension)
        self.norm2 = MinkowskiBatchNorm(planes, momentum=bn_momentum)
        self.conv3 = MinkowskiConvolution(planes, planes * 4, kernel_size=1, dimension=dimension)
        self.norm3 = MinkowskiBatchNorm(planes * 4, momentum=bn_momentum)
        self.relu = MinkowskiReLU(inplace=True)
        self.downsample = downsample

    def forward(self, x: SparseTensor) -> SparseTensor:
        out = conv_norm_act(self.conv1, self.norm1, ACT_RELU, x, training=self.training)
        out = conv_norm_act(self.conv2, self.norm2, ACT_RELU, out, training=self.training)
        if self.downsample is not None:
            r = self.downsample[0](x)
            residual = batch_norm_rows(r.F, self.downsample[1].bn, self.training)
        else:
            residual = x.F
        return conv_norm_act(self.conv3, self.norm3, ACT_RELU, out, res=residual, training=self.training)
