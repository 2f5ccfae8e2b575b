"""Every bf16 and fp32 kernel instance of the sparse branch of the training steps (MinkResNet + the FCAF3D head's sparse
layers), pinned per element against a float64 reference on the same operands (tests/bf16_bounds.py), at sizes derived from
the device's SM count so each case selects the instance it names. fp32 is the parity arithmetic: every fp32 sparse
convolution runs on the SIMT kernels and every fp32 normalisation on the centred two-pass esb_norm_fwd. Outputs are
pre-filled with NaN. Each case runs under torch.profiler and asserts that the instance it claims was launched; the census
test asserts that a C2-shaped bf16 step launches no sparse-branch instance outside the bf16 set (the fp32 steps are held
to the fp32 set by the whole-library census of test_head_elementwise_bf16_gpu.py)."""
import functools
import itertools
import json
import os
import re
import subprocess
import sys

import pytest
import torch

import bf16_bounds as B

pytestmark = pytest.mark.gpu
DEV = 'cuda:0'
BF = torch.bfloat16
F32 = torch.float32


def _bf(t, dtype=BF):
    return t.to(DEV, dtype).contiguous()


def _t(dtype):
    return '__nv_bfloat16' if dtype == BF else 'float'


def _out_rel(dtype):
    return B.OUT_REL_BF16 if dtype == BF else B.OUT_REL_F32


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


_INSTANCE = re.compile(r'(?<![\w])((?:spconv|norm|bn|seg|maxpool)_\w*(?:<[^<>()]*>)?)\(')
# The profiler runs in a fresh interpreter (sparse_bf16_child.py runs every case of this module there and fills this dict
# with {case label: launched instances}): in a process that has already run the model tests, short profiler sessions were
# seen to miss the first kernels they should record.
_CHILD = None


def _instances(fn):
    """(fn(), the set of sparse-branch kernel instances it launched, e.g. 'spconv_tc_fwd_kernel<256, 4, true>'); the set
    is only recorded in the child process."""
    if _CHILD is None:
        return fn(), set()
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        out = fn()
        torch.cuda.synchronize()
    seen = set()
    for e in prof.events():
        m = _INSTANCE.search(e.name)
        if m:
            seen.add(m.group(1))
    return out, seen


@functools.lru_cache(maxsize=None)
def _launched():
    p = subprocess.run([sys.executable, os.path.join(os.path.dirname(os.path.abspath(__file__)), 'sparse_bf16_child.py')],
                       capture_output=True, text=True, timeout=900)
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


# the instances each group of cases pins; the census test holds the C2 step to their union
TC_FWD = {(nt, mn): f'spconv_tc_fwd_kernel<{nt}, 4, {"true" if mn else "false"}>' for nt in (64, 128, 256) for mn in (1, 0)}
TC_WGRAD = {64: 'spconv_tc_wgrad_kernel<64, 4>', 128: 'spconv_tc_wgrad_kernel<128, 3>'}
TC_WGRAD_REDUCE = 'spconv_wgrad_reduce_kernel'
SIMT = ['spconv_fwd_kernel<__nv_bfloat16, false>', 'spconv_fwd_kernel<__nv_bfloat16, true>',
        'spconv_wgrad_kernel<__nv_bfloat16>']
NORM_STATS = ['seg_colstat_kernel<__nv_bfloat16, 0>', 'seg_colstat_kernel<__nv_bfloat16, 1>', 'seg_finalize_mean_kernel',
              'seg_finalize_rstd_kernel', 'norm_bwd_reduce_kernel<__nv_bfloat16>']
NORM_VEC8 = ['norm_apply_vec8_kernel<__nv_bfloat16>', 'norm_bwd_apply_vec8_kernel<__nv_bfloat16>']
NORM_SCALAR = ['norm_apply_kernel<__nv_bfloat16>', 'norm_bwd_apply_kernel<__nv_bfloat16>']
BN_FUSED = ['bn_stats_kernel<__nv_bfloat16>', 'bn_apply_fused_kernel<__nv_bfloat16>']
MAXPOOL = ['maxpool_fwd_kernel<__nv_bfloat16>', 'maxpool_bwd_kernel<__nv_bfloat16>']
PINNED = set(TC_FWD.values()) | set(TC_WGRAD.values()) | {TC_WGRAD_REDUCE} | set(SIMT) | set(NORM_STATS) | \
    set(NORM_VEC8) | set(NORM_SCALAR) | set(BN_FUSED) | set(MAXPOOL)
# fp32 (the parity arithmetic): SIMT convolutions at every width, esb_norm_fwd / esb_norm_bwd for every normalisation
SIMT_F32 = [s.replace('__nv_bfloat16', 'float') for s in SIMT]
NORM_STATS_F32 = [s.replace('__nv_bfloat16', 'float') for s in NORM_STATS]
NORM_VEC8_F32 = [s.replace('__nv_bfloat16', 'float') for s in NORM_VEC8]
NORM_SCALAR_F32 = [s.replace('__nv_bfloat16', 'float') for s in NORM_SCALAR]
MAXPOOL_F32 = [s.replace('__nv_bfloat16', 'float') for s in MAXPOOL]
PINNED_F32 = set(SIMT_F32) | set(NORM_STATS_F32) | set(NORM_VEC8_F32) | set(NORM_SCALAR_F32) | set(MAXPOOL_F32)


# ------------------------------------------------------------------------------------------------ tensor-core conv
# (N_TILE, cout of the call, cin of the call, row tiles as a function of the SM count)
_FWD_SHAPES = {256: (256, 128, lambda sms: sms), 128: (128, 192, lambda sms: sms), 64: (128, 64, lambda sms: sms // 2)}


@pytest.mark.parametrize('w_layout', [1, 0], ids=['fwd_MN', 'dgrad_K'])
@pytest.mark.parametrize('n_tile', [256, 128, 64])
def test_spconv_tc_fwd(n_tile, w_layout):
    """esb_spconv_tc_fwd: forward (w_layout 1: the stored (K, cin, cout) kernel) and dgrad (w_layout 0: (K, cout, cin)).
    The last row tile is partial; the middle tile has mask 0 (its rows must come out exactly zero); offset 5 has no
    neighbour and offset 7 exactly one."""
    from embodiedscan_b200 import sparse as SP
    from embodiedscan_b200._ffi import call, ptr, stream
    sms = _sms()
    cout, cin, tiles = _FWD_SHAPES[n_tile]
    n_out = 128 * tiles(sms) - 37
    assert B.tc_fwd_n_tile(n_out, cout, sms) == n_tile
    K, n_in = 27, n_out + 501
    gen = torch.Generator().manual_seed(n_tile + w_layout)
    nbr = B.random_kernel_map(n_in, n_out, K, gen, DEV, empty_offset=5, single_offset=7, empty_tile=tiles(sms) // 2)
    x = _bf(torch.randn(n_in, cin, generator=gen))
    wshape = (K, cin, cout) if w_layout else (K, cout, cin)
    w = _bf(torch.randn(wshape, generator=gen) / (K * cin) ** 0.5)
    masks = SP.KernelMap(nbr, n_in, n_out, K).tile_masks('out')
    assert int(masks[tiles(sms) // 2]) == 0 and (int(masks[0]) >> 5) & 1 == 0
    y = torch.full((n_out, cout), float('nan'), dtype=BF, device=DEV)

    def run():
        call('esb_spconv_tc_fwd', ptr(x), ptr(w), ptr(nbr), ptr(masks), ptr(y), n_out, cin, cout, K, w_layout, stream())
    _, seen = _instances(run)
    _claim(seen, [TC_FWD[(n_tile, w_layout)]], f'tc fwd N_TILE {n_tile} layout {w_layout}')
    ref, A, n_red = B.gather_gemm(x, w, nbr, w_layout)
    r = B.assert_within(y, ref, A, n_red, B.OUT_REL_BF16, 'tc fwd')
    print(f'ratio {r:.4g}')
    assert bool((y[(tiles(sms) // 2) * 128:(tiles(sms) // 2 + 1) * 128] == 0).all())
    B.assert_rejects(B.conv_faults(y, x, w, nbr, w_layout), ref, A, n_red, B.OUT_REL_BF16)


@pytest.mark.parametrize('cin,cout', [(192, 64), (256, 64), (192, 128), (256, 128)])
def test_spconv_tc_wgrad(cin, cout):
    """esb_spconv_tc_wgrad at n_tile 64 / 128 with a last A slice of 64 (cin 192) or 128 channels (cin 256). Offset 0 has no
    pair, offsets 1-3 have chunk_pairs - 1, chunk_pairs and chunk_pairs + 1 pairs, the others 1..3000. Into zeros, the
    result must equal, bit for bit, each pair chunk's gradient computed on its own (into zeros) added up in chunk order;
    into a non-zero dw0, the same chunk sum starting from dw0, and dw0 + gradient within the bound."""
    from embodiedscan_b200._ffi import call, ptr, stream
    sms = _sms()
    K, n_rows = 27, 3000
    hint = K * n_rows
    cp = B.tc_wgrad_chunk_pairs(hint, cin, cout, sms)
    gen = torch.Generator().manual_seed(cin + cout)
    counts = [0, cp - 1, cp, cp + 1] + [int(c) for c in torch.randint(1, n_rows + 1, (K - 4, ), generator=gen)]
    pin, pout, koff = B.random_pairs(counts, n_rows, n_rows, gen, DEV)
    koff_d = torch.tensor(koff, dtype=torch.int32, device=DEV)
    x = _bf(torch.randn(n_rows, cin, generator=gen))
    dy = _bf(torch.randn(n_rows, cout, generator=gen))

    def wgrad(dw, pi, po, ko, kk, h):
        call('esb_spconv_tc_wgrad', ptr(x), ptr(dy), ptr(pi), ptr(po), ptr(ko), ptr(dw), h, cin, cout, kk, stream())
        return dw

    g, seen = _instances(lambda: wgrad(torch.zeros((K, cin, cout), device=DEV), pin, pout, koff_d, K, hint))
    n_tile = 128 if cout % 128 == 0 else 64
    _claim(seen, [TC_WGRAD[n_tile], TC_WGRAD_REDUCE], f'tc wgrad cin {cin} cout {cout}')
    ref, A, n_red = B.pair_wgrad(x, dy, pin, pout, koff)
    r = B.assert_within(g, ref, A, n_red, B.OUT_REL_F32, 'tc wgrad')
    assert bool((g[0] == 0).all())
    B.assert_rejects(B.wgrad_faults(g, x, dy, pin, pout, koff, cp), ref, A, n_red, B.OUT_REL_F32)

    dw0 = torch.randn((K, cin, cout), generator=gen).to(DEV) * float(ref.abs().max()) / 4
    acc = wgrad(dw0.clone(), pin, pout, koff_d, K, hint)
    r = max(r, B.assert_within(acc, dw0.double() + ref, dw0.double().abs() + A, n_red + 1, B.OUT_REL_F32, 'tc wgrad dw0'))
    zero_sum, dw0_sum = torch.zeros_like(dw0), dw0.clone()
    n_multi = 0
    for k in range(K):
        starts = range(koff[k], koff[k + 1], cp)
        n_multi += len(starts) > 1
        for b in starts:
            e = min(b + cp, koff[k + 1])
            one = torch.tensor([0, e - b], dtype=torch.int32, device=DEV)
            part = wgrad(torch.zeros((1, cin, cout), device=DEV), pin[b:e], pout[b:e], one, 1, hint)[0]
            zero_sum[k] += part
            dw0_sum[k] += part
    assert n_multi >= 2, 'the chunk order is only visible on offsets with several chunks'
    assert torch.equal(g, zero_sum), 'chunk partials not added in chunk order'
    assert torch.equal(acc, dw0_sum), 'accumulating into a non-zero dw must add the chunks onto dw in chunk order'
    print(f'chunk_pairs {cp}, ratio {r:.4g}')


# ------------------------------------------------------------------------------------------------ SIMT conv
@pytest.mark.parametrize('cout', [64, 70])
@pytest.mark.parametrize('dtype', [BF, F32], ids=['bf16', 'fp32'])
def test_spconv_simt_stem(dtype, cout):
    """MinkResNet.conv1 (3 -> 64, k3 s2) runs on the SIMT kernels in bf16 and in fp32: forward, dgrad (the transposed-weight
    instance) and wgrad on the library's stride-2 kernel map. cout 70 is not a multiple of 4 (the scalar load path) nor of
    64."""
    from embodiedscan_b200 import sparse as SP
    from embodiedscan_b200._ffi import call, dtype_code, ptr, stream
    from oracle import sparse_ref as R
    import numpy as np
    g = np.random.RandomState(cout)
    c = np.concatenate([np.sort(g.randint(0, 2, (30000, 1)), 0), g.randint(-40, 40, (30000, 3))], 1)
    c = R.unique_first(c)[0]
    mgr = SP.CoordinateManager(DEV)
    key = mgr.insert_unique(torch.from_numpy(c).to(DEV, torch.int32), 1)
    km = mgr.kernel_map(key, mgr.stride_key(key, 2), 3)
    cin, K = 3, 27
    gen = torch.Generator().manual_seed(cout)
    x = _bf(torch.randn(km.n_in, cin, generator=gen), dtype)
    w = _bf(torch.randn(K, cin, cout, generator=gen) / (K * cin) ** 0.5, dtype)
    dy = _bf(torch.randn(km.n_out, cout, generator=gen), dtype)
    y = torch.full((km.n_out, cout), float('nan'), dtype=dtype, device=DEV)
    dx = torch.full((km.n_in, cin), float('nan'), dtype=dtype, device=DEV)
    dw = torch.zeros((K, cin, cout), device=DEV)
    pin, pout, koff, tot = km.pairs

    def run():
        code = dtype_code(dtype)
        call('esb_spconv_fwd', ptr(x), ptr(w), ptr(km.nbr_out), ptr(y), km.n_out, cin, cout, K, 0, code, stream())
        call('esb_spconv_fwd', ptr(dy), ptr(w), ptr(km.nbr_in), ptr(dx), km.n_in, cout, cin, K, 1, code, stream())
        call('esb_spconv_wgrad', ptr(x), ptr(dy), ptr(pin), ptr(pout), ptr(koff), ptr(dw), tot, cin, cout, K, code,
             stream())
    _, seen = _instances(run)
    _claim(seen, SIMT if dtype == BF else SIMT_F32, f'SIMT stem cout {cout}' + ('' if dtype == BF else ' fp32'))
    ref, A, n_red = B.gather_gemm(x, w, km.nbr_out, 1)
    # fp32: a 3-channel reduction through each of a few neighbours is too short to average its roundings (C_SHORT_F32)
    r1 = B.assert_within(y, ref, A, n_red, _out_rel(dtype), 'simt fwd', c=B.C_ACC if dtype == BF else B.C_SHORT_F32)
    ref, A, n_red = B.gather_gemm(dy, w, km.nbr_in, 0)
    r2 = B.assert_within(dx, ref, A, n_red, _out_rel(dtype), 'simt dgrad')
    ref, A, n_red = B.pair_wgrad(x, dy, pin, pout, koff.tolist())
    r3 = B.assert_within(dw, ref, A, n_red, B.OUT_REL_F32, 'simt wgrad')
    print(f'ratios fwd {r1:.4g} dgrad {r2:.4g} wgrad {r3:.4g}')


# (cin, cout) of the call: C1's cout 80 (not a multiple of the 64-channel tile), a cin that is not a multiple of the 16-channel
# reduction chunk, a cin and a cout that are not multiples of 4 (the scalar load4 path of x, of w and, in the dgrad, of dy),
# and C1's widest layer
SIMT_CASES = {'cin64_cout80': (64, 80), 'cin40_cout80': (40, 80), 'cin33_cout70': (33, 70), 'wide640': (640, 640)}


@pytest.mark.parametrize('exact', [False, True], ids=['random', 'exact'])
@pytest.mark.parametrize('w_layout', [1, 0], ids=['fwd', 'dgrad'])
@pytest.mark.parametrize('name', list(SIMT_CASES))
def test_spconv_simt_f32(name, w_layout, exact):
    """spconv_fwd_kernel<float, false> (forward: w (K, cin, cout)) and <float, true> (dgrad: w (K, cout, cin) read
    transposed), the 64 x 64 output tile with a 16-channel reduction chunk, into NaN. About sms / 2 row tiles, the last one
    partial; offset 5 has no neighbour, offset 7 exactly one, and the whole 64-row tile in the middle none (its rows must
    come out exactly 0). On operands in {-1, 0, 1} the fp32 sums are exact: bit for bit."""
    from embodiedscan_b200._ffi import call, dtype_code, ptr, stream
    cin, cout = SIMT_CASES[name]
    tiles = _sms() // 2
    n_out, K = 64 * tiles - 37, 27
    n_in = n_out + 501
    gen = torch.Generator().manual_seed(cin * 1000 + cout + 10 * w_layout + exact)
    nbr = B.random_kernel_map(n_in, n_out, K, gen, DEV, empty_offset=5, single_offset=7, empty_tile=tiles // 2,
                              tile_rows=64)
    wshape = (K, cin, cout) if w_layout else (K, cout, cin)
    if exact:
        d = min(0.5, (16.0 / (K * cin * 0.35)) ** 0.5)
        x, w = B.ternary((n_in, cin), d, gen), B.ternary(wshape, d, gen)
    else:
        x, w = torch.randn(n_in, cin, generator=gen), torch.randn(wshape, generator=gen) / (K * cin) ** 0.5
    x, w = _bf(x, F32), _bf(w, F32)
    y = torch.full((n_out, cout), float('nan'), dtype=F32, device=DEV)
    _, seen = _instances(lambda: call('esb_spconv_fwd', ptr(x), ptr(w), ptr(nbr), ptr(y), n_out, cin, cout, K,
                                      1 - w_layout, dtype_code(F32), stream()))
    _claim(seen, [SIMT_F32[1 - w_layout]], f'SIMT fp32 {name} layout {w_layout} {"exact" if exact else "random"}')
    ref, A, n_red = B.gather_gemm(x, w, nbr, w_layout)
    assert bool((y[(tiles // 2) * 64:(tiles // 2 + 1) * 64] == 0).all()), 'a tile without neighbours must be exactly 0'
    if exact:
        B.assert_exact(y, ref, A, f'simt {name}', out_bf16=False)
        return
    r = B.assert_within(y, ref, A, n_red, B.OUT_REL_F32, f'simt {name}')
    B.assert_rejects(B.conv_faults(y, x, w, nbr, w_layout, tile_rows=64, chunk=16), ref, A, n_red, B.OUT_REL_F32)
    print(f'ratio {r:.4g}')


# (cin, cout): splits > 1 at 64 x 64 (one tile per offset), splits > 1 with partial tiles and the scalar load path, and
# C1's widest layer, whose 27 x 100 tiles already fill the device (splits = 1)
SIMT_WGRAD_CASES = {'c64': (64, 64), 'cin40_cout70': (40, 70), 'wide640': (640, 640)}


@pytest.mark.parametrize('exact', [False, True], ids=['random', 'exact'])
@pytest.mark.parametrize('name', list(SIMT_WGRAD_CASES))
def test_spconv_simt_wgrad_f32(name, exact):
    """spconv_wgrad_kernel<float>: one partial of dW per pair split (bf16_bounds.simt_wgrad_splits), added in split order by
    the fixed-order finisher. Offset 0 has no pair, offset 1 fewer pairs than splits (the splits past its pairs write
    nothing), the others 1..3000. Into zeros, the result must equal, bit for bit, each split's gradient computed on its
    own (a one-offset call with one split) added in split order; into a non-zero dw0 the same chain starting from dw0; both
    within the bound (n_red = pairs + splits). On operands in {-1, 0, 1}: bit for bit against float64."""
    from embodiedscan_b200._ffi import call, dtype_code, ptr, stream
    cin, cout = SIMT_WGRAD_CASES[name]
    sms = _sms()
    K, n_rows = 27, 3000
    gen = torch.Generator().manual_seed(cin + cout + exact)
    counts = [0, 0] + [int(c) for c in torch.randint(1, n_rows + 1, (K - 2, ), generator=gen)]
    hint = sum(counts)
    splits = B.simt_wgrad_splits(hint, K, cin, cout, sms)
    assert (splits == 1) == (name == 'wide640'), splits
    counts[1] = max(splits - 1, 0)
    hint = sum(counts)
    assert B.simt_wgrad_splits(hint, K, cin, cout, sms) == splits
    pin, pout, koff = B.random_pairs(counts, n_rows, n_rows, gen, DEV)
    koff_d = torch.tensor(koff, dtype=torch.int32, device=DEV)
    if exact:
        d = (16.0 / n_rows) ** 0.5
        x, dy = B.ternary((n_rows, cin), d, gen), B.ternary((n_rows, cout), d, gen)
    else:
        x, dy = torch.randn(n_rows, cin, generator=gen), torch.randn(n_rows, cout, generator=gen)
    x, dy = _bf(x, F32), _bf(dy, F32)

    def wgrad(dw, pi, po, ko, kk, h):
        call('esb_spconv_wgrad', ptr(x), ptr(dy), ptr(pi), ptr(po), ptr(ko), ptr(dw), h, cin, cout, kk, dtype_code(F32),
             stream())
        return dw

    g, seen = _instances(lambda: wgrad(torch.zeros((K, cin, cout), device=DEV), pin, pout, koff_d, K, hint))
    _claim(seen, [SIMT_F32[2]], f'SIMT fp32 wgrad {name} {"exact" if exact else "random"}')
    ref, A, n_red = B.pair_wgrad(x, dy, pin, pout, koff)
    assert bool((g[0] == 0).all())
    if exact:
        B.assert_exact(g, ref, A, f'simt wgrad {name}', out_bf16=False)
    else:
        r = B.assert_within(g, ref, A, n_red + splits, B.OUT_REL_F32, 'simt wgrad')
        per = B.simt_wgrad_split_len(max(counts), splits)
        B.assert_rejects(B.wgrad_faults(g, x, dy, pin, pout, koff, per), ref, A, n_red + splits, B.OUT_REL_F32)
    dw0 = torch.randn((K, cin, cout), generator=gen).to(DEV) * max(float(ref.abs().max()), 1.0) / 4
    acc = wgrad(dw0.clone(), pin, pout, koff_d, K, hint)
    if not exact:
        r = max(r, B.assert_within(acc, dw0.double() + ref, dw0.double().abs() + A, n_red + splits + 1, B.OUT_REL_F32,
                                   'simt wgrad dw0'))
    zero_sum, dw0_sum = torch.zeros_like(dw0), dw0.clone()
    for k in range(K):
        n = koff[k + 1] - koff[k]
        per = B.simt_wgrad_split_len(n, splits)
        for s in range(splits):
            b, e = koff[k] + s * per, min(koff[k] + (s + 1) * per, koff[k + 1])
            if b >= e:
                continue
            one = torch.tensor([0, e - b], dtype=torch.int32, device=DEV)
            part = wgrad(torch.zeros((1, cin, cout), device=DEV), pin[b:e], pout[b:e], one, 1, 0)[0]
            zero_sum[k] += part
            dw0_sum[k] += part
    assert torch.equal(g, zero_sum), 'split partials not added in split order'
    assert torch.equal(acc, dw0_sum), 'accumulating into a non-zero dw must add the splits onto dw in split order'
    if not exact:
        print(f'splits {splits}, ratio {r:.4g}')


# ------------------------------------------------------------------------------------------------ normalisation
def _norm_case(sizes, C, res_too, gen, dtype=BF):
    N = sum(sizes)
    x = _bf(torch.randn(N, C, generator=gen) * 2 + 0.5, dtype)
    dy = _bf(torch.randn(N, C, generator=gen), dtype)
    res = _bf(torch.randn(N, C, generator=gen), dtype) if res_too else None
    gamma = torch.nn.Parameter((torch.rand(1, C, generator=gen) + 0.5).to(DEV))
    beta = torch.nn.Parameter(torch.randn(1, C, generator=gen).to(DEV))
    return x, dy, res, gamma, beta


def _check_norm(x, dy, res, gamma, beta, y, xg, sizes, eps, pivot, what, act=1):
    """Forward: ReLU and ELU are 1-Lipschitz, so the bound on z carries over to y. Backward, ReLU: the derivative read
    from the kernel's own y (a step: it must be the kernel's). ELU: the derivative e^z at the float64 z, and the kernel's
    y + 1 is off by at most the forward bound of y, which, times |dy|, is a `fixed` term carried through the backward
    formula (bf16_bounds.seg_norm_bwd_fixed). fp32 adds the documented error of rsqrtf and expm1f as fixed terms
    (bf16_bounds.seg_norm_fn_fixed)."""
    out_rel = _out_rel(x.dtype)
    f32 = x.dtype == F32
    z, A, n_red, st = B.seg_norm_ref(x, sizes, gamma.detach(), beta.detach(), eps, res, pivot)
    ya = B._act(z, act)
    F_y = B.seg_norm_fn_fixed(x, gamma.detach(), st, z, act) if f32 else 0.0
    r = B.assert_within(y, ya, A, n_red, out_rel, f'{what} fwd', fixed=F_y)
    F_dx = F_dg = F_db = 0.0
    if act == 1:
        gy = dy.double() * (y > 0)
    else:
        gy = dy.double() * torch.where(z > 0, 1.0, torch.exp(z))
        y_err = (out_rel * ya.abs() + B.C_ACC * B.U32 * n_red * A + F_y) * (1 + 2 * out_rel)
        F_dx, F_dg, F_db = B.seg_norm_bwd_fixed(x, dy.double().abs() * y_err, st)
        F_dx = F_dx * gamma.detach().double().abs().view(1, -1)
    if f32:
        _, f_dx, f_dg, f_db = B.seg_norm_fn_fixed(x, gamma.detach(), st, z, act, gy)
        F_dx, F_dg, F_db = F_dx + f_dx, F_dg + f_dg, F_db + f_db
    (dx, A_dx), (dg, A_dg), (db, A_db) = B.seg_norm_bwd_ref(x, gy, gamma.detach(), st)
    N = float(x.shape[0])
    r = max(r, B.assert_within(xg, dx, A_dx, n_red, out_rel, f'{what} dx', fixed=F_dx))
    r = max(r, B.assert_within(gamma.grad.view(-1), dg, A_dg, N, B.OUT_REL_F32, f'{what} dgamma', fixed=F_dg))
    r = max(r, B.assert_within(beta.grad.view(-1), db, A_db, N, B.OUT_REL_F32, f'{what} dbeta', fixed=F_db))
    return r


def _norm_claim(dtype, C):
    if dtype == F32:
        return NORM_STATS_F32 + (NORM_VEC8_F32 if C % 8 == 0 else NORM_SCALAR_F32)
    return NORM_STATS + (NORM_VEC8 if C % 8 == 0 else NORM_SCALAR)


@pytest.mark.parametrize('act', [1, 2], ids=['relu', 'elu'])
@pytest.mark.parametrize('C', [64, 12])
@pytest.mark.parametrize('dtype', [BF, F32], ids=['bf16', 'fp32'])
def test_instance_norm(dtype, C, act):
    """MinkowskiInstanceNorm + ReLU / ELU in bf16 and fp32 (esb_norm_fwd / esb_norm_bwd with one segment per scan): 4 scans
    of unequal size, one spanning three 256-row statistics blocks. C = 12 takes the non-vec8 apply kernels."""
    from embodiedscan_b200 import sparse as SP
    gen = torch.Generator().manual_seed(C)
    sizes = [700, 37, 258, 129]
    x, dy, _, gamma, beta = _norm_case(sizes, C, False, gen, dtype)
    seg_off = torch.tensor([0] + list(itertools.accumulate(sizes)), dtype=torch.int32, device=DEV)
    row_seg = torch.repeat_interleave(torch.arange(4), torch.tensor(sizes)).to(DEV, torch.int32)
    xg = x.clone().requires_grad_(True)

    def run():
        y = SP.seg_norm(xg, gamma, beta, seg_off, row_seg, 4, max(sizes), 1e-8, act)
        y.backward(dy)
        return y
    y, seen = _instances(run)
    _claim(seen, _norm_claim(dtype, C), f'instance norm C {C} act {act}' + ('' if dtype == BF else ' fp32'))
    r = _check_norm(x, dy, None, gamma, beta, y.detach(), xg.grad, sizes, 1e-8, False, 'instance norm', act)
    print(f'ratio {r:.4g}')


@pytest.mark.parametrize('act', [1, 2], ids=['relu', 'elu'])
@pytest.mark.parametrize('C,N', [(8, 3001), (2048, 517), (12, 1001)])
@pytest.mark.parametrize('dtype', [BF, F32], ids=['bf16', 'fp32'])
def test_batch_norm(dtype, C, N, act):
    """BatchNorm + residual + ReLU / ELU on the training path. bf16: the fused single-pass kernels at their shared-memory
    edges C = 8 (256 rows per step) and C = 2048 (one row per step), and the esb_norm_fwd fallback at C = 12 (not a
    multiple of 8); the pivot row is offset from the mean to exercise the shifted statistics. fp32 (the parity arithmetic)
    takes the centred two-pass esb_norm_fwd at every C. Backward through esb_norm_bwd."""
    from embodiedscan_b200 import sparse as SP
    torch.manual_seed(C)
    gen = torch.Generator().manual_seed(C)
    x, dy, res, _, _ = _norm_case([N], C, True, gen, dtype)
    x[0] += 3.0
    bn = torch.nn.BatchNorm1d(C).to(DEV)
    with torch.no_grad():
        bn.weight.uniform_(0.5, 1.5)
        bn.bias.normal_()
    xg = x.clone().requires_grad_(True)

    def run():
        y = SP.batch_norm_rows(xg, bn, True, act, res)
        y.backward(dy)
        return y
    y, seen = _instances(run)
    fused = C % 8 == 0 and dtype == BF
    _claim(seen, BN_FUSED + [NORM_STATS[-1], NORM_VEC8[1]] if fused else _norm_claim(dtype, C),
           f'batch norm C {C} act {act}' + ('' if dtype == BF else ' fp32'))
    r = _check_norm(x, dy, res, bn.weight, bn.bias, y.detach(), xg.grad, [N], bn.eps, fused, 'batch norm', act)
    print(f'ratio {r:.4g}')


# ------------------------------------------------------------------------------------------------ max pooling
@pytest.mark.parametrize('C', [64, 12])
@pytest.mark.parametrize('dtype', [BF, F32], ids=['bf16', 'fp32'])
def test_maxpool_ties(dtype, C):
    """Sparse k2 s2 max pooling in bf16 and fp32 on values from {-2, ..., 2} (most windows tie). Forward: bit-equal to the
    oracle. Backward: each output's gradient goes to exactly one input, the one through the LOWEST kernel offset among the
    tied maxima (maxpool_fwd_kernel keeps the first maximum: `v > best`)."""
    from embodiedscan_b200 import sparse as SP
    from oracle import sparse_ref as R
    import numpy as np
    g = np.random.RandomState(C)
    c = np.concatenate([np.sort(g.randint(0, 2, (20000, 1)), 0), g.randint(-8, 8, (20000, 3))], 1)   # dense windows
    c = R.unique_first(c)[0]
    mgr = SP.CoordinateManager(DEV)
    key = mgr.insert_unique(torch.from_numpy(c).to(DEV, torch.int32), 1)
    mgr.batch_size = 2
    gen = torch.Generator().manual_seed(C)
    x = _bf(torch.randint(-2, 3, (c.shape[0], C), generator=gen).float(), dtype)
    xg = x.clone().requires_grad_(True)
    pool = SP.MinkowskiMaxPooling()

    def run():
        t = pool(SP.SparseTensor(xg, coordinate_map_key=key, coordinate_manager=mgr))
        return t
    t, seen = _instances(lambda: run().F)
    km = mgr.kernel_map(key, mgr.stride_key(key, 2), 2)
    nbr = km.nbr_out.cpu().numpy().astype(np.int64)
    assert np.array_equal(nbr, R.kernel_map(c, R.unique_first(c, 2)[0], R.offsets(2, 1)))
    assert torch.equal(t.cpu(), R.maxpool(x.float().cpu(), nbr).to(dtype))
    dy = _bf(torch.randn(km.n_out, C, generator=gen), dtype)
    _, seen_b = _instances(lambda: t.backward(dy))
    _claim(seen | seen_b, MAXPOOL if dtype == BF else MAXPOOL_F32, f'max pool C {C}' + ('' if dtype == BF else ' fp32'))
    # expected gradient: lowest offset among the tied maxima
    nb = km.nbr_out.long()
    vals = torch.where((nb >= 0)[:, :, None], x.float()[nb.clamp(min=0)], torch.tensor(float('-inf'), device=DEV))
    top = vals.max(0).values
    is_max = vals == top[None]
    k_star = torch.argmax(is_max.to(torch.int8), 0)           # the first maximal index along the offsets
    rows = nb[k_star, torch.arange(km.n_out, device=DEV)[:, None]]   # (n_out, C): nb[k_star[o, c], o]
    assert int((is_max.sum(0) > 1).sum()) > km.n_out * C // 4, 'the inputs must tie often'
    ref = torch.zeros((km.n_in, C), dtype=dtype, device=DEV)
    ref[rows, torch.arange(C, device=DEV)[None].expand_as(rows)] = dy
    assert torch.equal(xg.grad, ref)


# ------------------------------------------------------------------------------------------------ census
def test_c2_step_launches_only_pinned_instances():
    """One C2-shaped bf16 forward + backward (the synth batch of test_c2_shaped_bf16_step_matches_oracle) under the
    profiler: every sparse-branch kernel instance it launches (spconv*, norm*, bn_*, seg_*, and the sparse maxpool_*) must
    be one the cases above pin. A change that makes the step select a new instance fails here until a case pins it."""
    if _CHILD is None:
        seen = _claim(set(), [], 'C2 bf16 step')
    else:
        from embodiedscan_b200 import MODELS
        from embodiedscan_b200.synth import mv_det3d_config, synth_batch
        torch.manual_seed(0)
        model = MODELS.build(dict(mv_det3d_config('C2'), compute_dtype=BF)).to(DEV).train()
        batch = synth_batch(7, 1, n_views=20, H=480, W=640, n_points=100000, augment=True)

        def step():
            data = model.data_preprocessor(dict(inputs=batch['inputs'], data_samples=batch['data_samples']), True)
            losses = model(**data, mode='loss')
            sum(losses.values()).backward()
        seen = _claim(_instances(step)[1], [], 'C2 bf16 step')
    assert seen, 'the profiler saw no sparse-branch kernel'
    assert seen <= PINNED, f'instances no case pins: {sorted(seen - PINNED)}'
