"""The head, loss and elementwise kernels of the bf16 and fp32 training steps, pinned per element against a float64
reference on the same operands (tests/bf16_bounds.py) or bit for bit, and one census over the whole library: every library
kernel a C2, C3 or C4 bf16 training step (C2 with its optimiser step) or a C1 (with its optimiser step), C3 or C4 fp32
training step launches is pinned here, in test_sparse_bf16_gpu.py or in test_dense_bf16_gpu.py, or is named in EXACT with
the test that holds it bit for bit or to a fixture.

  * focal_fwd_kernel / focal_bwd_kernel (fp32 and bf16 logits): the loss sum and the per-element gradient against mmcv's
    formula in float64 (bf16_bounds.focal_ref, whose conditioning factor K(x) = 1 + e^|x| is part of the element term),
    on 'typical' head logits, on logits uniform in [-12, 12], and at the C2 size (~444k block partials through the
    ordered finisher; the textbook bound of that sum is too loose to see a single-row fault there, so its faults are
    checked on the smaller cases). Saturated logits (x <= -89, where expf overflows; x >= 17, where p rounds to 1) against
    mmcv's clamp to log(FLT_MIN) in closed form.
  * bias_act_kernel / act_bwd_kernel: the 2-D backbone's epilogue, in place as backbones._BiasResAct calls it.
  * gather2_rows_kernel, img_normalize_kernel (bf16 and fp32), cast_kernel<bf16>: bit for bit.
  * interp_features_kernel: multilinear interpolation against float64 on the same features (an 11-term bound).
  * backbones._BiasResAct's bias gradient: a ResNet with a trainable BN affine in eval mode (norm_eval with the default
    norm_cfg) against a float64 restatement, fp32 and bf16, through the CUDA graph and without it.

Worst ratios measured on an H100 SXM (80 GB HBM3, 132 SMs, 700 W power limit), c = C_ACC = 0.5 throughout: focal 0.0667,
bias_act 0.284, act_bwd 0.367 (its `fixed` term carries the rest), interp 0.152; bf16_bounds.py's docstring has the
details, and the fp32 ratios of the sparse and dense modules.

Each case runs under torch.profiler in a fresh interpreter (head_elementwise_bf16_child.py) and claims the instances it
launched, as the sparse and dense modules do."""
import ast
import ctypes
import functools
import glob
import json
import os
import re
import subprocess
import sys
from unittest import mock

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import bf16_bounds as B

pytestmark = pytest.mark.gpu
DEV = 'cuda:0'
BF = torch.bfloat16
F32 = torch.float32
NAN = float('nan')
HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(os.path.dirname(HERE), 'embodiedscan_b200', 'csrc')
_CHILD = None


# ------------------------------------------------------------------------------------------------ the library's kernels
@functools.lru_cache(maxsize=None)
def library_kernels():
    """Every kernel name the library declares, parsed from the `__global__` declarations of csrc/*.cu."""
    pat = re.compile(r'__global__\s+(?:static\s+)?void\s+(?:__launch_bounds__\([^)]*\)\s*)?(\w+)\s*\(')
    names = set()
    for f in glob.glob(os.path.join(CSRC, '*.cu')):
        with open(f) as fh:
            names.update(pat.findall(fh.read()))
    return frozenset(names)


def library_instance(event_name, lib=None):
    """The instance ('name<args>' or 'name') of a profiler kernel event if it is one of the library's kernels, else None.
    Only unqualified names or names in the anonymous namespace count: at::native::...fill_kernel is not hash.cu's."""
    lib = library_kernels() if lib is None else lib
    s = event_name[5:] if event_name.startswith('void ') else event_name
    if s.startswith('(anonymous namespace)::'):
        s = s[len('(anonymous namespace)::'):]
    m = re.match(r'[A-Za-z_]\w*', s)
    if not m or m.group(0) not in lib:
        return None
    j = m.end()
    if s[j:j + 1] == '<':
        depth = 0
        for j in range(m.end(), len(s)):
            depth += {'<': 1, '>': -1}.get(s[j], 0)
            if depth == 0:
                break
        j += 1
    return s[:j] if s[j:j + 1] == '(' else None


def _instances(fn):
    """(fn(), the library kernel instances it launched); the set is only recorded in the child process."""
    if _CHILD is None:
        return fn(), set()
    from torch.profiler import ProfilerActivity, profile
    for _ in range(5):      # a short profiler session was seen to record no kernel at all: then record the case again
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            out = fn()
            torch.cuda.synchronize()
        seen = {i for i in map(library_instance, (e.name for e in prof.events())) if i}
        if seen:
            break
    return out, seen


@functools.lru_cache(maxsize=None)
def _launched():
    env = dict(os.environ, ESB200_TEXT_RANDOM_INIT='1')
    p = subprocess.run([sys.executable, os.path.join(HERE, 'head_elementwise_bf16_child.py')], capture_output=True,
                       text=True, timeout=900, env=env)
    rows = [json.loads(l) for l in p.stdout.splitlines() if l.startswith('{')]
    assert p.returncode == 0 and rows, (p.returncode, p.stderr[-2000:])
    return rows[-1]


def _claim(seen, claimed, what):
    """Assert that case `what` launched every instance in `claimed`; returns the instances it launched."""
    if _CHILD is not None:
        _CHILD[what] = sorted(seen)
        return seen
    seen = set(_launched().get(what, ()))
    print(f'{what}: launched {sorted(seen)}')
    missing = set(claimed) - seen
    assert not missing, f'{what}: expected {sorted(missing)} among the launched instances {sorted(seen)}'
    return seen


def _t(dtype):
    return '__nv_bfloat16' if dtype == BF else 'float'


FOCAL = [f'focal_{d}_kernel<{t}>' for d in ('fwd', 'bwd') for t in ('float', '__nv_bfloat16')]
BIAS_ACT = [f'bias_act_kernel<{t}>' for t in ('float', '__nv_bfloat16')]
ACT_BWD = [f'act_bwd_kernel<{t}>' for t in ('float', '__nv_bfloat16')]
GATHER2 = [f'gather2_rows_kernel<{t}>' for t in ('float', '__nv_bfloat16')]
INTERP = [f'interp_features_kernel<{t}>' for t in ('float', '__nv_bfloat16')]
IMG_NORM = 'img_normalize_kernel<__nv_bfloat16>'
IMG_NORM_F32 = 'img_normalize_kernel<float>'
CAST = 'cast_kernel<__nv_bfloat16>'
PINNED = set(FOCAL) | set(BIAS_ACT) | set(ACT_BWD) | set(GATHER2) | set(INTERP) | {IMG_NORM, IMG_NORM_F32, CAST}


# ------------------------------------------------------------------------------------------------ focal loss
def _focal(x, t, w, gamma, alpha, scale):
    """esb_focal_loss_fwd into a zeroed sum and esb_focal_loss_bwd into a NaN-filled gradient."""
    from embodiedscan_b200._ffi import call, dtype_code, ptr, stream
    n, C = x.shape
    total = torch.zeros(1, dtype=F32, device=DEV)
    s = torch.tensor([scale], dtype=F32, device=DEV)
    grad = torch.full_like(x, NAN)
    call('esb_focal_loss_fwd', ptr(x), ptr(t), n, C, gamma, alpha, ptr(w), ptr(total), dtype_code(x.dtype), stream())
    call('esb_focal_loss_bwd', ptr(x), ptr(t), n, C, gamma, alpha, ptr(w), ptr(s), ptr(grad), dtype_code(x.dtype), stream())
    return total[0], grad


# name: (rows, C, wide logits, fault checks)
FOCAL_CASES = {'c284': (3001, 284, False, True), 'c1': (1001, 1, False, True), 'wide284': (3001, 284, True, False),
               'c2_size': (400001, 284, False, False)}


@pytest.mark.parametrize('name,dtype', [(n, d) for n in FOCAL_CASES for d in (F32, BF) if n != 'c2_size' or d == BF],
                         ids=lambda v: {F32: 'fp32', BF: 'bf16'}.get(v, v))
def test_focal_loss(name, dtype):
    """The loss sum and the per-element gradient (scale 0.37) against mmcv's formula in float64; targets -1, in range
    and >= C; unequal row weights, the last row heavy (so the last, partial, block of the sum matters). The C2-size case
    runs the bf16 instance, the one the C2 step launches."""
    n, C, wide, faults = FOCAL_CASES[name]
    gen = torch.Generator().manual_seed(n + C + wide)
    x, t, w = B.focal_operands(n, C, gen, wide)
    x, t, w = x.to(DEV, dtype), t.to(DEV), w.to(DEV)
    gamma, alpha, scale = 2.0, 0.25, 0.37
    (total, grad), seen = _instances(lambda: _focal(x, t, w, gamma, alpha, scale))
    _claim(seen, [f'focal_fwd_kernel<{_t(dtype)}>', f'focal_bwd_kernel<{_t(dtype)}>', 'sum_partial_rows_kernel'],
           f'focal {name} {dtype}')
    ref = B.focal_ref(x, t, w, gamma, alpha, scale)
    n_blocks = (n * C + 255) // 256
    val, A = B.focal_sum_bound(ref, n_blocks)
    r = B.assert_within(total, val, A, 1, B.OUT_REL_F32, f'focal {name} sum')
    out_rel = B.OUT_REL_BF16 if dtype == BF else B.OUT_REL_F32
    Ag = ref['K'] * ref['g'].abs()
    r = max(r, B.assert_within(grad, ref['g'], Ag, B.FOCAL_ELEM, out_rel, f'focal {name} grad'))
    if faults:
        B.assert_rejects(B.focal_faults_fwd(x, t, w, gamma, alpha, total), val, A, 1, B.OUT_REL_F32)
    if name != 'c2_size':
        B.assert_rejects(B.focal_faults_bwd(x, t, w, gamma, alpha, scale, grad), ref['g'], Ag, B.FOCAL_ELEM, out_rel)
    print(f'ratio {r:.4g}')


@pytest.mark.parametrize('dtype', [F32, BF], ids=['fp32', 'bf16'])
def test_focal_loss_saturated(dtype):
    """Logits where the fp32 sigmoid saturates: x <= -89 (expf(-x) overflows, p = 0) and x >= 17 (1 + expf(-x) rounds to
    1, p = 1). mmcv clamps the log's argument to FLT_MIN, so a positive at p = 0 costs alpha (-log FLT_MIN) and has
    gradient -alpha, a negative at p = 1 costs (1 - alpha)(-log FLT_MIN) with gradient 1 - alpha, and the other two
    combinations are exactly zero; times row weight and scale (powers of two here, so the closed forms are exact but for
    log(FLT_MIN)). Each value within 1 ulp of the closed form; the sum within the bound of its additions."""
    gen = torch.Generator().manual_seed(89)
    n, C = 777, 13
    sat = torch.tensor([-89.0, -100.0, -1000.0, 17.0, 20.0, 100.0])
    x = sat[torch.randint(0, 6, (n, C), generator=gen)]
    t = torch.randint(-1, C + 2, (n, ), generator=gen)
    w = 2.0 ** -torch.randint(0, 6, (n, ), generator=gen).float()
    x, t, w = x.to(DEV, dtype), t.to(DEV), w.to(DEV)
    gamma, alpha, scale = 2.0, 0.25, 0.5
    (total, grad), seen = _instances(lambda: _focal(x, t, w, gamma, alpha, scale))
    _claim(seen, [f'focal_fwd_kernel<{_t(dtype)}>', f'focal_bwd_kernel<{_t(dtype)}>'], f'focal saturated {dtype}')
    pos = t.view(-1, 1) == torch.arange(C, device=DEV).view(1, -1)
    lo, hi = x.double() <= -89, x.double() >= 17
    wd = w.double().view(-1, 1)
    l = torch.where(pos & lo, -alpha * B.LOG_FLT_MIN, 0.0) + torch.where(~pos & hi, -(1 - alpha) * B.LOG_FLT_MIN, 0.0)
    g = torch.where(pos & lo, -alpha, 0.0) + torch.where(~pos & hi, 1 - alpha, 0.0)
    g = g * wd * scale
    assert bool((pos & lo).any()) and bool((~pos & hi).any()) and bool((pos & hi).any()) and bool((~pos & lo).any())
    ulp = lambda v, dt: torch.finfo(dt).eps * 2.0 ** torch.floor(torch.log2(v.abs().clamp(min=1e-30)))  # noqa: E731
    assert bool(((grad.double() - g).abs() <= ulp(g, dtype) * (g != 0)).all()), 'saturated gradient'
    l = l * wd
    val, A = l.sum(), (5 + 8 + (n * C + 255) // 256) * l.abs().sum()
    B.assert_within(total, val, A, 1, B.OUT_REL_F32, 'saturated loss sum')
    for xv, tv, want in ((-89.0, 0, -alpha * B.LOG_FLT_MIN), (-1000.0, 0, -alpha * B.LOG_FLT_MIN),
                         (17.0, -1, -(1 - alpha) * B.LOG_FLT_MIN), (100.0, 3, -(1 - alpha) * B.LOG_FLT_MIN),
                         (17.0, 0, 0.0), (-89.0, 1, 0.0)):
        one, _ = _focal(torch.tensor([[xv]], device=DEV, dtype=dtype), torch.tensor([tv], device=DEV),
                        torch.ones(1, device=DEV), gamma, alpha, scale)
        bound = float(ulp(torch.tensor(want, dtype=torch.float64), F32)) if want else 0.0
        assert abs(float(one) - want) <= bound, (xv, tv, float(one), want)


# ------------------------------------------------------------------------------------------------ bias + act epilogue
def _bias_act(x, bias, res, y, act):
    from embodiedscan_b200._ffi import call, dtype_code, ptr, stream
    call('esb_bias_act_fwd', ptr(x), ptr(bias), ptr(res), ptr(y), x.shape[0], x.shape[1], act, dtype_code(x.dtype),
         stream())
    return y


@pytest.mark.parametrize('res', [False, True], ids=['nores', 'res'])
@pytest.mark.parametrize('C', [8, 2048])
@pytest.mark.parametrize('act', [0, 1, 2], ids=['none', 'relu', 'elu'])
@pytest.mark.parametrize('dtype', [F32, BF], ids=['fp32', 'bf16'])
def test_bias_act(dtype, act, C, res):
    """esb_bias_act_fwd in place (y == x, as backbones._BiasResAct calls it) on random operands against float64, with a
    number of 8-channel pieces that is not a multiple of the 256-thread block (C = 8) and one row per block (C = 2048);
    out of place into NaN on operands in {-2..2} with an integer bias, where the fp32 sums are exact (act none / ReLU:
    bit for bit)."""
    rows = 1001 if C == 8 else 37
    gen = torch.Generator().manual_seed(C + act + 10 * res)
    x = torch.randn(rows, C, generator=gen).to(DEV, dtype)
    b = torch.randn(C, generator=gen).to(DEV)
    r = torch.randn(rows, C, generator=gen).to(DEV, dtype) if res else None
    xi = torch.randint(-2, 3, (rows, C), generator=gen).to(DEV, dtype)
    bi = torch.randint(-3, 4, (C, ), generator=gen).float().to(DEV)
    ri = torch.randint(-2, 3, (rows, C), generator=gen).to(DEV, dtype) if res else None
    y = x.clone()
    ye = torch.full_like(xi, NAN)

    def run():
        _bias_act(y, b, r, y, act)
        _bias_act(xi, bi, ri, ye, act)
    _, seen = _instances(run)
    _claim(seen, [f'bias_act_kernel<{_t(dtype)}>'], f'bias act {dtype} {act} C {C} res {res}')
    out_rel = B.OUT_REL_BF16 if dtype == BF else B.OUT_REL_F32
    ref, A, n_red = B.bias_act_ref(x, b, r, act)
    ratio = B.assert_within(y, ref, A, n_red, out_rel, 'bias act')
    B.assert_rejects(B.bias_act_faults(y, x, b, r, act, 256 * 8 // C), ref, A, n_red, out_rel)
    ref, A, n_red = B.bias_act_ref(xi, bi, ri, act)
    if act < 2:
        assert torch.equal(ye.double(), ref), 'integer operands: the sums are exact'
    else:
        ratio = max(ratio, B.assert_within(ye, ref, A, n_red, out_rel, 'bias act ELU integer'))
    print(f'ratio {ratio:.4g}')


@pytest.mark.parametrize('n', [8 * 3001 + 5, 8 * 2048], ids=['tail', 'whole'])
@pytest.mark.parametrize('act', [1, 2], ids=['relu', 'elu'])
@pytest.mark.parametrize('dtype', [F32, BF], ids=['fp32', 'bf16'])
def test_act_bwd(dtype, act, n):
    """esb_act_bwd (dx = dy act'(y), the derivative read from the stored output y) against the derivative at the float64
    pre-activation z, into NaN: n % 8 != 0 takes the scalar tail. z has exact zeros (ReLU at y = 0 exactly: derivative 0)
    and values down to -20 (ELU at y = -1 in bf16: y + 1 = 0 against e^z). Reading the derivative from the rounded y is
    bf16_bounds.act_bwd_ref's `fixed` term; the case prints the c the bound would need without it."""
    from embodiedscan_b200._ffi import call, dtype_code, ptr, stream
    gen = torch.Generator().manual_seed(n + act)
    z = torch.randn(n, generator=gen, dtype=torch.float64) * 3
    z[::7] = 0.0
    z[3::11] = -20.0 + torch.rand(z[3::11].shape, generator=gen, dtype=torch.float64) * 5
    y = B._act(z, act).to(dtype).to(DEV)
    z = z.to(DEV)
    dy = torch.randn(n, generator=gen).to(DEV, dtype)
    dx = torch.full_like(dy, NAN)
    _, seen = _instances(lambda: call('esb_act_bwd', ptr(dy), ptr(y), ptr(dx), n, act, dtype_code(dtype), stream()))
    _claim(seen, [f'act_bwd_kernel<{_t(dtype)}>'], f'act bwd {dtype} {act} n {n}')
    out_rel = B.OUT_REL_BF16 if dtype == BF else B.OUT_REL_F32
    ref, A, n_red, fixed = B.act_bwd_ref(dy, z, y, act)
    r = B.assert_within(dx, ref, A, n_red, out_rel, 'act bwd', fixed=fixed)
    at0 = z == 0
    assert bool((dx[at0] == (0 if act == 1 else dy[at0])).all()), 'the derivative at y = 0 (ReLU: 0, ELU: 1)'
    hidden = B.excess_ratio(dx, ref, A, n_red, out_rel)              # the c the fixed term would need inside c
    B.assert_rejects(B.act_bwd_faults(dx, dy, z, act), ref, A, n_red, out_rel, fixed)
    print(f'ratio {r:.4g}, without the fixed term {hidden:.4g}')


# ------------------------------------------------------------------------------------------------ row gather
@pytest.mark.parametrize('mode', ['ia_null', 'ia_neg_b_null', 'both_neg'])
@pytest.mark.parametrize('C', [8, 1024])
@pytest.mark.parametrize('dtype', [F32, BF], ids=['fp32', 'bf16'])
def test_gather2_rows(dtype, C, mode):
    """esb_gather2_rows, bit for bit against torch indexing and one fp32 addition per element (one rounding): ia NULL
    (identity on the first na < n rows), explicit ia with negative entries, b / ib NULL, negative ib; into NaN."""
    from embodiedscan_b200._ffi import call, dtype_code, ptr, stream
    gen = torch.Generator().manual_seed(C + len(mode))
    n, na, nb = 1337, 900, 1100
    a = torch.randn(na, C, generator=gen).to(DEV, dtype)
    b = torch.randn(nb, C, generator=gen).to(DEV, dtype)
    ia = None if mode == 'ia_null' else torch.randint(-300, na, (n, ), generator=gen).to(torch.int32).to(DEV)
    ib = None if mode == 'ia_neg_b_null' else torch.randint(-400, nb, (n, ), generator=gen).to(torch.int32).to(DEV)
    bb = None if ib is None else b
    out = torch.full((n, C), NAN, dtype=dtype, device=DEV)
    _, seen = _instances(lambda: call('esb_gather2_rows', ptr(a), ptr(ia), na, ptr(bb), ptr(ib), ptr(out), n, C,
                                      dtype_code(dtype), stream()))
    _claim(seen, [f'gather2_rows_kernel<{_t(dtype)}>'], f'gather2 {dtype} C {C} {mode}')
    rows_a = torch.where(torch.arange(n, device=DEV) < na, torch.arange(n, device=DEV), -1) if ia is None else ia.long()
    ref = torch.where((rows_a >= 0)[:, None], a.float()[rows_a.clamp(min=0)], 0.0)
    if ib is not None:
        ref = ref + torch.where((ib >= 0)[:, None], b.float()[ib.long().clamp(min=0)], 0.0)
        assert bool((ib < 0).any())
    assert bool((rows_a < 0).any())
    assert torch.equal(out, ref.to(dtype))


# ------------------------------------------------------------------------------------------------ interpolation
@pytest.mark.parametrize('ts', [1, 2, 8])
@pytest.mark.parametrize('C', [1, 18, 128])
@pytest.mark.parametrize('dtype', [F32, BF], ids=['fp32', 'bf16'])
def test_interp_features(dtype, C, ts):
    """esb_interp_features through SparseTensor.features_at_coordinates (integer queries) against float64 multilinear
    interpolation on the same features: negative coordinates (the floor), queries on lattice points (one weight exactly
    1), corners absent from the lattice; 11 terms (eight products and additions, the three roundings of a weight)."""
    from embodiedscan_b200 import sparse as SP
    g = np.random.RandomState(C * 10 + ts)
    c = np.concatenate([g.randint(0, 2, (3000, 1)), g.randint(-9, 9, (3000, 3)) * ts], 1)
    c = np.unique(c, axis=0)
    c = c[g.permutation(c.shape[0])]
    q = np.concatenate([g.randint(0, 2, (2000, 1)), g.randint(-10 * ts, 10 * ts, (2000, 3))], 1)
    q[:300] = c[:300]                                                    # on lattice points
    mgr = SP.CoordinateManager(DEV)
    mgr.batch_size = 2
    key = mgr.insert_unique(torch.from_numpy(c).to(DEV, torch.int32), ts)
    feats = torch.from_numpy(g.randn(c.shape[0], C)).to(DEV, dtype)
    cm = mgr.maps[key]
    rows_lib = cm.coords.cpu().numpy().astype(np.int64)                  # the lattice's own row order
    st = SP.SparseTensor(feats, coordinate_map_key=key, coordinate_manager=mgr)
    qd = torch.from_numpy(q).to(DEV, torch.int32)
    out, seen = _instances(lambda: st.features_at_coordinates(qd))
    _claim(seen, [f'interp_features_kernel<{_t(dtype)}>'], f'interp {dtype} C {C} ts {ts}')
    ref, A, n_red, rows, wt = B.interp_ref(rows_lib, feats, ts, q)
    assert bool((rows < 0).any()) and bool((rows[:300, 0] >= 0).all()) and bool((wt[:300, 0] == 1).all())
    r = B.assert_within(out, ref, A, n_red, B.OUT_REL_F32, 'interp')
    faults = B.interp_faults(out, rows_lib, feats, ts, q)
    B.assert_rejects(faults if ts > 1 else faults[2:], ref, A, n_red, B.OUT_REL_F32)
    print(f'ratio {r:.4g}')


# ------------------------------------------------------------------------------------------------ bit-exact elementwise
@pytest.mark.parametrize('bgr', [0, 1])
@pytest.mark.parametrize('channels_last', [0, 1])
@pytest.mark.parametrize('dtype', [BF, F32], ids=['bf16', 'fp32'])
def test_img_normalize(dtype, channels_last, bgr):
    """esb_img_normalize to bf16 and fp32, bit for bit against CPU ((px - mean) / std) in fp32 (for bf16 then rounded to
    bf16: the same double rounding), on several images with H < Hp and W < Wp (the padding exactly zero), into NaN."""
    from embodiedscan_b200._ffi import call, dtype_code, ptr, stream
    g = torch.Generator().manual_seed(channels_last * 2 + bgr)
    n, H, W, Hp, Wp = 3, 37, 45, 64, 64
    src = torch.randint(0, 256, (n, 3, H, W), generator=g, dtype=torch.uint8)
    mean, std = [123.675, 116.28, 103.53], [58.395, 57.12, 57.375]
    m3, s3 = (ctypes.c_float * 3)(*mean), (ctypes.c_float * 3)(*std)
    shape = (n, Hp, Wp, 3) if channels_last else (n, 3, Hp, Wp)
    dst = torch.full(shape, NAN, dtype=dtype, device=DEV)
    sd = src.to(DEV)
    _, seen = _instances(lambda: call('esb_img_normalize', ptr(sd), n, H, W, Hp, Wp, ctypes.cast(m3, ctypes.c_void_p),
                                      ctypes.cast(s3, ctypes.c_void_p), bgr, channels_last, ptr(dst), dtype_code(dtype),
                                      stream()))
    _claim(seen, [IMG_NORM if dtype == BF else IMG_NORM_F32],
           f'img normalize cl {channels_last} bgr {bgr}' + ('' if dtype == BF else ' fp32'))
    px = src.float()[:, [2, 1, 0]] if bgr else src.float()
    v = ((px - torch.tensor(mean).view(1, 3, 1, 1)) / torch.tensor(std).view(1, 3, 1, 1)).float().to(dtype)
    ref = torch.zeros((n, 3, Hp, Wp), dtype=dtype)
    ref[:, :, :H, :W] = v
    got = dst.cpu().permute(0, 3, 1, 2) if channels_last else dst.cpu()
    assert torch.equal(got, ref)
    assert bool((got[:, :, H:] == 0).all() and (got[:, :, :, W:] == 0).all())


def test_cast_f32_to_bf16():
    """esb_cast_f32_to_bf16 bit for bit against tensor.to(torch.bfloat16): +-0, fp32 subnormals, exact ties (round half to
    even, both parities), values rounding up to +-inf, +-inf and random values; NaN stays NaN (the payload may differ)."""
    from embodiedscan_b200._ffi import call, ptr, stream
    bits = [0x00000000, 0x80000000, 0x00000001, 0x807FFFFF, 0x00400000, 0x00008000, 0x00018000,   # zeros, subnormals
            0x3F808000, 0x3F818000, 0xBF808000, 0xBF818000,                                      # ties to even
            0x7F7FFFFF, 0xFF7FFFFF, 0x7F7F8000, 0x7F7F7FFF, 0x7F800000, 0xFF800000,               # up to inf, inf
            0x7FC00000, 0xFFC00001, 0x7F800001]                                                  # NaNs
    g = torch.Generator().manual_seed(1)
    special = torch.tensor(bits, dtype=torch.int64).to(torch.int32).view(torch.float32)
    x = torch.cat([special, torch.randn(1001, generator=g) * 10.0 ** torch.randint(-40, 38, (1001, ), generator=g)])
    xd = x.to(DEV)
    out = torch.full(x.shape, NAN, dtype=BF, device=DEV)
    _, seen = _instances(lambda: call('esb_cast_f32_to_bf16', ptr(xd), ptr(out), x.numel(), stream()))
    _claim(seen, [CAST], 'cast')
    ref = x.to(BF)
    o = out.cpu()
    nan = torch.isnan(ref)
    assert torch.equal(torch.isnan(o), nan)
    assert torch.equal(o[~nan].view(torch.int16), ref[~nan].view(torch.int16)), 'bits differ (signed zeros included)'


# ------------------------------------------------------------------------------------------------ _BiasResAct
def _rel(got, want):
    return float((got.double() - want).norm() / want.norm())


def _resnet_ref(net, x):
    """The ResNet of backbones.py restated in float64: conv2d, the eval-mode BN formula on its running statistics,
    residual, ReLU; returns (outputs, {name: leaf tensor}) with a float64 leaf per conv weight and BN affine parameter."""
    leaves = {}
    for name, p in net.named_parameters():
        leaves[name] = p.detach().double().requires_grad_(p.requires_grad)

    def cb(prefix, m, x, relu, res=None):
        w, gam, bet = leaves[prefix + '.conv.weight'], leaves[prefix + '.bn.weight'], leaves[prefix + '.bn.bias']
        bn = m.bn
        y = F.conv2d(x, w, None, m.conv.stride, m.conv.padding)
        scale = gam / torch.sqrt(bn.running_var.double() + bn.eps)
        y = y * scale.view(1, -1, 1, 1) + (bet - bn.running_mean.double() * scale).view(1, -1, 1, 1)
        y = y + res if res is not None else y
        return F.relu(y) if relu else y
    y = F.max_pool2d(cb('stem', net.stem, x, True), 3, 2, 1)
    outs = []
    for i in range(net.num_stages):
        for j, blk in enumerate(getattr(net, f'layer{i + 1}')):
            p = f'layer{i + 1}.{j}'
            idt = cb(p + '.ds', blk.ds, y, False) if blk.ds is not None else y
            y = cb(p + '.cb2', blk.cb2, cb(p + '.cb1', blk.cb1, y, True), True, res=idt)
        outs.append(y)
    return outs, leaves


@pytest.mark.parametrize('mode', ['fp32', 'bf16_graphed', 'bf16_eager'])
def test_trainable_bn_affine_gets_its_gradient(mode):
    """ResNet(depth=18, base_channels=16, frozen_stages=1, norm_eval=True) with the default norm_cfg: the BatchNorms of
    stages 2-4 are in eval mode with a trainable affine, so their folded shift beta - mean * scale requires grad and the
    conv's bias + residual + ReLU runs through backbones._BiasResAct. The gradients of every trainable BN weight and bias
    (and, off the graph, of the input) must match a float64 restatement: bn.bias gets sum(g) over N, H, W, and bn.weight
    the -running_mean d(shift) part. Running statistics and affine are random, as after training. bf16 runs through the
    CUDA-graphed backbone and with ESB200_GRAPH2D=0; the graph's captured callable is given an input without grad. At the
    parent of this test's commit bn.bias.grad was None."""
    from embodiedscan_b200.backbones import ResNet
    torch.manual_seed(3)
    dtype = F32 if mode == 'fp32' else BF
    net = ResNet(depth=18, base_channels=16, frozen_stages=1, norm_eval=True)
    gen = torch.Generator().manual_seed(4)
    with torch.no_grad():
        for m in net.modules():
            if isinstance(m, torch.nn.BatchNorm2d):
                m.weight.uniform_(0.5, 1.5, generator=gen)
                m.bias.normal_(generator=gen)
                m.running_mean.normal_(0, 0.5, generator=gen)
                m.running_var.uniform_(0.5, 2.0, generator=gen)
            if isinstance(m, torch.nn.Conv2d) and dtype == BF:
                m.weight.copy_(m.weight.bfloat16().float())
    net = net.to(DEV).train()
    trainable = [n for n, p in net.named_parameters() if p.requires_grad and '.bn.' in n]
    assert trainable and all(not n.startswith(('stem', 'layer1')) for n in trainable)
    x = torch.randn(2, 3, 64, 96, generator=gen).to(DEV, dtype).contiguous(memory_format=torch.channels_last)
    graphed = mode == 'bf16_graphed'
    xg = x.clone().requires_grad_(not graphed)
    dys = None

    def run():
        nonlocal dys
        with mock.patch.dict(os.environ, {'ESB200_GRAPH2D': '1' if graphed else '0'}):
            assert net._graphable(xg) == graphed
            outs = net(xg)
        dys = [torch.randn(o.shape, generator=gen).to(DEV) for o in outs]
        sum((o.float() * d).sum() for o, d in zip(outs, dys)).backward()
    _, seen = _instances(run)
    if not graphed:
        _claim(seen, [f'bias_act_kernel<{_t(dtype)}>', f'act_bwd_kernel<{_t(dtype)}>'], f'resnet trainable bn {mode}')
    x_ref = x.double().requires_grad_(not graphed)
    outs, leaves = _resnet_ref(net, x_ref)
    sum((o * d.double()).sum() for o, d in zip(outs, dys)).backward()
    params = dict(net.named_parameters())
    # fp32 holds the arithmetic element by element (at the parent commit it failed: bn.bias.grad was None). bf16 rounds
    # the folded filters, every activation and every gradient through the stages, and a BN parameter's gradient is a sum
    # of either sign over those (a weight's over cin k^2 filter taps, a bias's over N H W pixels): on an H100 the relative
    # 2-norm errors reached 0.164 (fp32: 0.001). The bf16 cases hold the two bf16 paths, through the CUDA graph and
    # without it, to 0.25
    rtol = 0.25
    for n in trainable:
        got, want = params[n].grad, leaves[n].grad
        assert got is not None and bool(got.abs().max() > 0), f'{n}: no gradient'
        if dtype == F32:
            err = float((got.double() - want).abs().max())
            assert err <= 1e-2 * float(want.abs().max()), f'{n}: max error {err:.3g} of {float(want.abs().max()):.3g}'
        else:
            err = float((got.double() - want).norm() / want.norm())
            assert err <= rtol, f'{n}: relative 2-norm error {err:.3g}'
    if not graphed:
        err = float((xg.grad.double() - x_ref.grad).norm() / x_ref.grad.norm())
        assert err <= (1e-3 if dtype == F32 else rtol), f'input gradient: relative 2-norm error {err:.3g}'
    print(f'{mode}: largest relative 2-norm error {max(_rel(params[n].grad, leaves[n].grad) for n in trainable):.3g}')


# ------------------------------------------------------------------------------------------------ census
# Library kernels held bit for bit or to a fixture rather than by a per-element bound: {kernel: the test that holds it}.
EXACT = {
    'voxelize_kernel': 'test_kernels_gpu.py::test_voxelize_bit_exact',
    'hash_clear_kernel': 'test_kernels_gpu.py::test_coord_unique_bit_exact',
    'hash_insert_min_kernel': 'test_kernels_gpu.py::test_coord_unique_bit_exact',
    'flag_winner_kernel': 'test_kernels_gpu.py::test_coord_unique_bit_exact',
    'compact_winner_kernel': 'test_kernels_gpu.py::test_coord_unique_bit_exact',
    'inverse_map_kernel': 'test_kernels_gpu.py::test_coord_unique_bit_exact',
    'hash_build_kernel': 'test_kernels_gpu.py::test_kernel_map_bit_exact',
    'hash_lookup_kernel': 'test_kernels_gpu.py::test_kernel_map_bit_exact',
    'kernel_map_kernel': 'test_kernels_gpu.py::test_kernel_map_bit_exact',
    'kernel_map_transpose_kernel': 'test_kernels_gpu.py::test_kernel_map_bit_exact',
    'fill_kernel': 'test_kernels_gpu.py::test_kernel_map_bit_exact',
    'pair_flag_kernel': 'test_kernels_gpu.py::test_kernel_map_bit_exact',
    'pair_compact_kernel': 'test_kernels_gpu.py::test_kernel_map_bit_exact',
    'generative_children_kernel': 'test_kernels_gpu.py::test_generative_and_union_bit_exact',
    'tile_mask_kernel': 'test_sparse_bf16_gpu.py::test_spconv_tc_fwd',
    'count_inside_kernel': 'test_kernels_gpu.py::test_fcaf3d_targets_bit_exact',
    'best_level_kernel': 'test_kernels_gpu.py::test_fcaf3d_targets_bit_exact',
    'topk_threshold_kernel': 'test_kernels_gpu.py::test_fcaf3d_targets_bit_exact',
    'count_scan_points_kernel': 'test_kernels_gpu.py::test_fcaf3d_targets_bit_exact',
    'assign_kernel': 'test_kernels_gpu.py::test_fcaf3d_targets_bit_exact',
    'bbox_cd_loss_kernel': 'test_losses_gpu.py::test_detector_head_fused_box_loss_matches_reference',
    'chamfer_nn_kernel': 'test_losses_gpu.py::test_chamfer_distance_matches_reference',
    'chamfer_keys_kernel': 'test_losses_gpu.py::test_chamfer_distance_matches_reference',
    'chamfer_grad_kernel': 'test_losses_gpu.py::test_chamfer_distance_matches_reference',
    'rotated_iou3d_fwd_kernel': 'test_rotiou_gpu.py::test_kernel_matches_float64_oracle_on_random_pairs',
    'rotated_iou3d_bwd_kernel': 'test_rotiou_gpu.py::test_head_losses_and_gradient_match_reference',
    'hungarian_kernel': 'test_kernels_gpu.py::test_hungarian_batch_equals_scipy',
    'box3d_overlap_kernel': 'test_kernels_gpu.py::test_box3d_overlap_9dof',
    'sum_partial_rows_kernel': 'test_partial_sum_gpu.py::test_sum_partial_rows_bit_exact',
    'sumsq_kernel': 'test_optim_gpu.py::test_grouped_adamw_kernel_matches_float64',
    'clip_coef_kernel': 'test_optim_gpu.py::test_grouped_adamw_kernel_matches_float64',
    'adamw_kernel': 'test_optim_gpu.py::test_grouped_adamw_kernel_matches_float64',
    'depth_flag_kernel': 'test_kernels_gpu.py::test_unproject_depth',
    'unproject_kernel': 'test_kernels_gpu.py::test_unproject_depth',
}


def _pinned_everywhere():
    import test_dense_bf16_gpu as D
    import test_sparse_bf16_gpu as S
    return S.PINNED | S.PINNED_F32 | D.PINNED | D.PINNED_F32 | PINNED


def unheld(seen, pinned, exact):
    """The launched instances neither pinned nor (by kernel name) in `exact`."""
    return sorted(i for i in seen if i not in pinned and i.split('<')[0] not in exact)


def test_exact_table_names_existing_tests():
    """Every test EXACT names exists (a test function of that name in that module)."""
    for kernel, where in EXACT.items():
        path, fn = where.split('::')
        with open(os.path.join(HERE, path)) as fh:
            names = {n.name for n in ast.walk(ast.parse(fh.read())) if isinstance(n, ast.FunctionDef)}
        assert fn in names, f'{kernel}: {where} does not exist'
        assert kernel in library_kernels(), f'{kernel} is not a library kernel'
    assert not set(EXACT) & {i.split('<')[0] for i in _pinned_everywhere()}, 'a kernel both pinned and in EXACT'


test_exact_table_names_existing_tests.no_child = True


# the census steps: bf16 C2 (with its optimiser step), C3, C4; fp32 (the parity arithmetic) C1 (with its optimiser step),
# C3, C4
CENSUS = ['C2', 'C3', 'C4', 'C1-fp32', 'C3-fp32', 'C4-fp32']


def _census_label(variant):
    name, _, dt = variant.partition('-')
    return f'{name} {dt or "bf16"} step, whole library'


@pytest.mark.parametrize('variant', CENSUS)
def test_step_launches_only_held_library_kernels(variant):
    """One training forward + backward of C2 (with the OptimWrapper step: cast, clip and AdamW), C3 and C4 in bf16, and of
    C1 (with its OptimWrapper step), C3 and C4 in fp32, on the census batches of test_dense_bf16_gpu.py: every library
    kernel instance launched must be pinned (here, or in the sparse or dense module) or, by kernel name, held bit for bit
    or to a fixture by the test EXACT names."""
    name, _, dt = variant.partition('-')
    with_optim = name in ('C1', 'C2')
    if _CHILD is None:
        seen = _claim(set(), [], _census_label(variant))
    else:
        import test_dense_bf16_gpu as D
        from embodiedscan_b200.engine import OptimWrapper
        model, batch = D.census_step(name, F32 if dt == 'fp32' else BF)
        optim = OptimWrapper(model) if with_optim else None

        def step():
            data = model.data_preprocessor(dict(inputs=batch['inputs'], data_samples=batch['data_samples']), True)
            loss = sum(model(**data, mode='loss').values())
            optim.update_params(loss) if optim is not None else loss.backward()
        seen = _claim(_instances(step)[1], [], _census_label(variant))
    assert len(seen) > 20, f'the profiler saw only {sorted(seen)}'
    if variant == 'C2':
        assert CAST in seen, 'the optimiser step was not recorded'
    if with_optim:
        assert any(i.split('<')[0] == 'adamw_kernel' for i in seen), 'the optimiser step was not recorded'
    bad = unheld(seen, _pinned_everywhere(), EXACT)
    assert not bad, f'library kernels no test holds: {bad}'


def test_census_rule_names_what_it_misses():
    """Dropping any one entry of the pinned sets or of EXACT makes the rule fail with that kernel's name, on the
    instances the bf16 and fp32 census steps launched."""
    rec = _launched()
    seen = set().union(*(rec.get(_census_label(v), ()) for v in CENSUS))
    pinned = _pinned_everywhere()
    assert not unheld(seen, pinned, EXACT)
    for inst in sorted(seen & pinned):
        assert unheld(seen, pinned - {inst}, EXACT) == [inst] or inst.split('<')[0] in EXACT
    for k in sorted({i.split('<')[0] for i in seen} & set(EXACT)):
        missing = unheld(seen, pinned, {e: v for e, v in EXACT.items() if e != k})
        assert missing and all(m.split('<')[0] == k for m in missing), (k, missing)


test_census_rule_names_what_it_misses.no_child = True


def test_library_instance_rule():
    """Only unqualified names and names in the anonymous namespace are the library's."""
    lib = frozenset({'fill_kernel', 'focal_fwd_kernel', 'sum_partial_rows_kernel'})
    assert library_instance('void (anonymous namespace)::fill_kernel(int*, long long, int)', lib) == 'fill_kernel'
    assert library_instance('void focal_fwd_kernel<__nv_bfloat16>(__nv_bfloat16 const*, long long const*)', lib) == \
        'focal_fwd_kernel<__nv_bfloat16>'
    assert library_instance('void at::native::fill_kernel<float>(float*)', lib) is None
    assert library_instance('void at::native::vectorized_elementwise_kernel<4, at::native::FillFunctor<float> >(int)',
                            lib) is None
    assert library_instance('sum_partial_rows_kernel(float const*, int, long long, float*, int, int)', lib) == \
        'sum_partial_rows_kernel'
    assert library_instance('void cub::DeviceScanKernel<int>(int)', lib) is None
    assert len(library_kernels()) > 70


test_library_instance_rule.no_child = True
