"""Every bf16 and fp32 kernel instance of the dense branch of the training steps (the per-view image backbone, point
painting, the occupancy Conv3d neck, the grounding attention), pinned per element against a float64 reference on the same
operands (tests/bf16_bounds.py), at sizes derived from the device's SM count so each case reaches the geometry it names.
fp32 is the parity arithmetic: every fp32 2-D convolution runs on the SIMT direct kernels (conv2d_direct.cu), all three
passes, and painting runs its fp32 instances. Outputs are pre-filled with NaN: an element no CTA writes fails. Each conv case also runs on operands in {-1, 0, 1}, where the result
must equal the reference bit for bit however long the reduction; the split sums (conv wgrad, attention dQ) are checked
to be added in split order, bit for bit. Each case runs under torch.profiler (in a fresh interpreter, see
dense_bf16_child.py) and asserts that the instance it claims was launched; the census tests assert that the C2, C3 and
C4 steps launch no dense-branch instance outside that set."""
import functools
import json
import os
import re
import subprocess
import sys

import pytest
import torch
import torch.nn.functional as F

import bf16_bounds as B

pytestmark = pytest.mark.gpu
DEV = 'cuda:0'
BF = torch.bfloat16
F32 = torch.float32
NAN = float('nan')


def _t(dtype):
    return '__nv_bfloat16' if dtype == BF else 'float'


def _out_rel(dtype):
    return B.OUT_REL_BF16 if dtype == BF else B.OUT_REL_F32


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


_INSTANCE = re.compile(r'(?<![\w])((?:conv_tma|conv2d_direct|stem7x7|maxpool2d|attn|paint)_\w*(?:<[^<>()]*>)?)\(')
_CHILD = None


def _instances(fn):
    """(fn(), the set of dense-branch kernel instances it launched); the set is only recorded in the child process."""
    if _CHILD is None:
        return fn(), set()
    from torch.profiler import ProfilerActivity, profile
    for _ in range(3):      # a short profiler session was seen to record no kernel at all: then record the case again
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            out = fn()
            torch.cuda.synchronize()
        seen = {m.group(1) for m in map(_INSTANCE.search, (e.name for e in prof.events())) if m}
        if seen:
            break
    return out, seen


@functools.lru_cache(maxsize=None)
def _launched():
    env = dict(os.environ, ESB200_TEXT_RANDOM_INIT='1')
    p = subprocess.run([sys.executable, os.path.join(os.path.dirname(os.path.abspath(__file__)), 'dense_bf16_child.py')],
                       capture_output=True, text=True, timeout=900, env=env)
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


def CONV(n, mn):
    return f'conv_tma_kernel<{n}, {"true" if mn else "false"}>'


def WGRAD(n):
    return f'conv_tma_wgrad_kernel<{n}>'


STEM = 'stem7x7_tc_kernel'
DIRECT_FWD, DIRECT_DGRAD = 'conv2d_direct_fwd_kernel<__nv_bfloat16>', 'conv2d_direct_dgrad_kernel<__nv_bfloat16>'
POOL = {8: 'maxpool2d_nhwc_kernel<__nv_bfloat16, 8>', 1: 'maxpool2d_nhwc_kernel<__nv_bfloat16, 1>'}
ATTN = ['attn_fwd_kernel', 'attn_delta_kernel', 'attn_bwd_kernel']
PAINT = ['paint_fwd_kernel<__nv_bfloat16>', 'paint_bwd_pairs_kernel<__nv_bfloat16>', 'paint_bwd_sum_kernel<__nv_bfloat16>']
PINNED = {CONV(n, mn) for n in (16, 32, 64, 128) for mn in (False, True)} | {WGRAD(n) for n in (16, 32, 64, 128)} | \
    {STEM, DIRECT_FWD, DIRECT_DGRAD} | set(POOL.values()) | set(ATTN) | set(PAINT)
DIRECT_FWD_F32, DIRECT_DGRAD_F32 = 'conv2d_direct_fwd_kernel<float>', 'conv2d_direct_dgrad_kernel<float>'
DIRECT_WGRAD_F32 = 'conv2d_direct_wgrad_kernel<float>'
POOL_F32 = 'maxpool2d_nhwc_kernel<float, 1>'
PAINT_F32 = [s.replace('__nv_bfloat16', 'float') for s in PAINT]
PINNED_F32 = {DIRECT_FWD_F32, DIRECT_DGRAD_F32, DIRECT_WGRAD_F32, POOL_F32} | set(PAINT_F32)


# ------------------------------------------------------------------------------------------------ calls
def _cl(t):
    """(N, C, *S) -> the kernels' channels-last memory (N, *S, C), contiguous."""
    return t.movedim(1, -1).contiguous()


def _nan(shape, dtype=BF):
    return torch.full(shape, NAN, dtype=dtype, device=DEV)


def _out_size(S, k, stride, pad):
    return [(s + 2 * pad - k) // stride + 1 for s in S]


def _fwd(x, w, bias, res, stride, pad, relu):
    """esb_conv{2,3}d_tma_fwd: x (N, Cin, *S) bf16, w (Cout, Cin, *k) bf16 -> (N, Cout, *So) written into NaN."""
    from embodiedscan_b200._ffi import call, ptr, stream
    N, cin, *S = x.shape
    cout, k = w.shape[0], w.shape[2]
    y = _nan([N, *_out_size(S, k, stride, pad), cout])
    xc, wc, rc = _cl(x), _cl(w), _cl(res) if res is not None else None
    if len(S) == 2:
        call('esb_conv2d_tma_fwd', ptr(xc), ptr(wc), ptr(bias), ptr(rc), ptr(y), N, *S, cin, cout, k, k, stride, pad,
             int(relu), stream())
    else:
        call('esb_conv3d_tma_fwd', ptr(xc), ptr(wc), ptr(bias), ptr(rc), ptr(y), N, *S, cin, cout, k, stride, pad,
             int(relu), stream())
    return y.movedim(-1, 1)


def _dgrad(dy, w, x_shape, stride, pad):
    from embodiedscan_b200._ffi import call, ptr, stream
    N, cin, *S = x_shape
    cout, k = w.shape[0], w.shape[2]
    dx = _nan([N, *S, cin])
    dyc, wc = _cl(dy), _cl(w)
    if len(S) == 2:
        call('esb_conv2d_tma_dgrad', ptr(dyc), ptr(wc), ptr(dx), N, *S, cin, cout, k, k, stride, pad, stream())
    else:
        call('esb_conv3d_tma_dgrad', ptr(dyc), ptr(wc), ptr(dx), N, *S, cin, cout, k, stride, pad, stream())
    return dx.movedim(-1, 1)


def _wgrad(x, dy, w_shape, stride, pad, dw0=None):
    """esb_conv{2,3}d_tma_wgrad into dw0 (Cout, Cin, *k) fp32 (zeros if None): the entry points ADD the gradient."""
    from embodiedscan_b200._ffi import call, ptr, stream
    N, cin, *S = x.shape
    cout, k, dims = w_shape[0], w_shape[2], len(w_shape) - 2
    perm = (dims + 1, dims) + tuple(range(dims))                 # (*k, Cin, Cout) -> (Cout, Cin, *k)
    inv = tuple(perm.index(i) for i in range(dims + 2))
    dw_t = (torch.zeros(w_shape, device=DEV) if dw0 is None else dw0).permute(inv).contiguous()
    xc, dyc = _cl(x), _cl(dy)
    if dims == 2:
        call('esb_conv2d_tma_wgrad', ptr(xc), ptr(dyc), ptr(dw_t), N, *S, cin, cout, k, k, stride, pad, stream())
    else:
        call('esb_conv3d_tma_wgrad', ptr(xc), ptr(dyc), ptr(dw_t), N, *S, cin, cout, k, stride, pad, stream())
    return dw_t.permute(perm)


# ------------------------------------------------------------------------------------------------ TMA conv cases
# (dims, cin, cout, k, stride, pad, spatial extent, residual, images: an int, or None = the fewest images giving some
# CTA >= 2 output tiles, a partial last tile and (wgrad) >= 2 pixel-tile splits)
CONV_CASES = {
    'n16_3x3_res': (2, 16, 16, 3, 1, 1, (37, 45), True, None),       # 32B swizzle, 4 taps per stage, 9 taps: last stage 1/4
    'n32_3x3_s2': (2, 32, 32, 3, 2, 1, (61, 83), False, None),       # 64B swizzle, element strides, odd extent
    'n64_tn': (2, 64, 64, 3, 1, 1, (3, 3), True, None),              # 128B swizzle, whole small images per tile (TN > 1)
    'n128_c1024': (2, 1024, 256, 1, 1, 0, (17, 19), True, None),     # 16 channel chunks per tap, two channel blocks
    'n128_c2048': (2, 2048, 256, 1, 1, 0, (17, 19), False, None),    # 32 chunks (C3's layer4 / FPN input width)
    'n128_co2048': (2, 512, 2048, 1, 1, 0, (17, 19), True, None),    # 16 channel blocks (C3's layer4 expansion)
    'n16_1x1_s2': (2, 64, 16, 1, 2, 0, (31, 41), False, None),       # 1x1 / stride 2: the dgrad memset
    'n16_tn': (2, 16, 16, 3, 1, 1, (3, 3), False, None),             # TN > 1 at every N_TILE, forward and dgrad
    'n32_tn_res': (2, 32, 32, 3, 1, 1, (3, 3), True, None),
    'n128_tn': (2, 128, 128, 3, 1, 1, (3, 3), True, None),
    'n64_s2_res': (2, 64, 64, 3, 2, 1, (33, 47), True, None),        # N_TILE 64 forward with element strides
    '3d_td': (3, 64, 64, 3, 1, 1, (11, 3, 5), False, None),          # TD > 1, partial along depth
    '3d_s2': (3, 64, 128, 3, 2, 1, (13, 21, 25), False, None),         # eight parity classes of unequal size
    '3d_neck_c3': (3, 768, 128, 3, 1, 1, (8, 10, 10), False, 1),     # C3's neck input width
    # carried over from the earlier tolerance-of-the-maximum checks
    'old_1x1_sq': (2, 64, 16, 1, 1, 0, (30, 40), False, 3),
    'old_3x3_16': (2, 16, 16, 3, 1, 1, (30, 40), False, 3),
    'old_expand_res': (2, 16, 64, 1, 1, 0, (30, 40), True, 3),
    'old_3x3_32_odd': (2, 32, 32, 3, 1, 1, (17, 23), False, 2),
    'old_3x3_64': (2, 64, 64, 3, 1, 1, (30, 40), False, 2),
    'old_3x3_128_tn': (2, 128, 128, 3, 1, 1, (15, 20), False, 5),
    'old_1x1_s2_ds': (2, 64, 128, 1, 2, 0, (30, 40), False, 2),
    'old_3x3_s2_odd': (2, 32, 32, 3, 2, 1, (31, 41), False, 2),
    'old_n256_res': (2, 256, 512, 1, 1, 0, (15, 20), True, 4),
    'old_8chunks': (2, 512, 128, 1, 1, 0, (15, 20), False, 4),
    'old_many_tiles': (2, 16, 16, 1, 1, 0, (120, 160), False, 2),
    'old3d_64': (3, 64, 64, 3, 1, 1, (6, 10, 8), False, 2),
    'old3d_s2': (3, 64, 128, 3, 2, 1, (6, 10, 8), False, 2),
    'old3d_1x1_s2': (3, 128, 256, 1, 2, 0, (6, 10, 8), False, 1),
    'old3d_256': (3, 256, 256, 3, 1, 1, (4, 5, 5), False, 1),
    'old3d_768': (3, 768, 256, 3, 1, 1, (4, 6, 5), False, 1),
}


# cases whose output tiles (forward and stride-1 dgrad) and wgrad boxes hold several whole images
TN_CASES = {'n16_tn', 'n32_tn_res', 'n64_tn', 'n128_tn'}


def _pixels(dims, S, n):
    return (n, ) + ((1, ) if dims == 2 else ()) + tuple(S)


@functools.lru_cache(maxsize=None)
def _images(name, sms):
    dims, cin, cout, k, stride, pad, S, res, n = CONV_CASES[name]
    if n is not None:
        return n
    So = _out_size(S, k, stride, pad)
    for n in range(1, 4096):
        g = B.conv_tma_geometry(*_pixels(dims, So, n), cout, sms)
        wg = B.wgrad_tma_geometry(*_pixels(dims, So, n), cin, cout, k ** dims, sms)
        short = wg['last_split'] < wg['tiles_per_cta'] or name not in WGRAD_SPLIT_CASES
        if g['per_cta'] >= 2 and g['partial'] and wg['n_splits'] >= 2 and short:
            return n
    raise AssertionError(name)


def _operands(name, exact, gen):
    dims, cin, cout, k, stride, pad, S, res, n = CONV_CASES[name]
    n = _images(name, _sms())
    taps = k ** dims
    xs, ws = (n, cin, *S), (cout, cin) + (k, ) * dims
    So = _out_size(S, k, stride, pad)
    ys = (n, cout, *So)
    if exact:       # expected partial sum ~ 16 (A <= 2^11 is asserted)
        d = min(0.5, (16.0 / (taps * cin)) ** 0.5)
        x, w = B.ternary(xs, d, gen), B.ternary(ws, d, gen)
        bias = torch.randint(-4, 5, (cout, ), generator=gen).float()
        r = torch.randint(-4, 5, ys, generator=gen).float() if res else None
        dd = min(0.5, (16.0 / (taps * cout)) ** 0.5)
        dy = B.ternary(ys, dd, gen)
        dw_d = min(0.5, (512.0 / (n * So[0] * So[1] * (So[2] if dims == 3 else 1))) ** 0.5)
        x_w, dy_w = B.ternary(xs, dw_d, gen), B.ternary(ys, dw_d, gen)
    else:
        x, w = torch.randn(xs, generator=gen), torch.randn(ws, generator=gen) / (taps * cin) ** 0.5
        bias = torch.randn(cout, generator=gen)
        r = torch.randn(ys, generator=gen) if res else None
        dy = torch.randn(ys, generator=gen)
        x_w, dy_w = x, dy
    bf = lambda t: t.to(DEV, BF) if t is not None else None  # noqa: E731
    return dict(x=bf(x), w=bf(w), bias=bias.to(DEV), res=bf(r), dy=bf(dy), x_w=bf(x_w), dy_w=bf(dy_w), n=n)


@pytest.mark.parametrize('exact', [False, True], ids=['random', 'exact'])
@pytest.mark.parametrize('name', list(CONV_CASES))
def test_conv_tma(name, exact):
    """conv_tma_kernel forward (fused bias + residual + ReLU) and dgrad, and conv_tma_wgrad_kernel (accumulating into a
    non-zero dw), per element against float64 torch convolutions; bit for bit on operands in {-1, 0, 1}."""
    dims, cin, cout, k, stride, pad, S, res, _ = CONV_CASES[name]
    sms = _sms()
    gen = torch.Generator().manual_seed(sum(map(ord, name)) + exact)
    o = _operands(name, exact, gen)
    n, taps = o['n'], k ** dims
    So = _out_size(S, k, stride, pad)
    g = B.conv_tma_geometry(*_pixels(dims, So, n), cout, sms)
    wg = B.wgrad_tma_geometry(*_pixels(dims, So, n), cin, cout, taps, sms)
    if CONV_CASES[name][-1] is None:
        assert g['per_cta'] >= 2 and g['partial'] and wg['n_splits'] >= 2
    if name in TN_CASES:
        assert g['tile'][3] > 1 and wg['box'][3] > 1, (g['tile'], wg['box'])
        assert B.conv_tma_geometry(*_pixels(dims, S, n), cin, sms)['tile'][3] > 1
    do_dgrad = stride in (1, 2) and (cin <= 256 and cin & (cin - 1) == 0 or cin % 256 == 0)
    x, w, wshape = o['x'], o['w'], (cout, cin) + (k, ) * dims
    dw0 = None if exact else torch.randn(wshape, generator=gen).to(DEV)

    def run():
        y = _fwd(x, w, o['bias'], o['res'], stride, pad, True)
        dx = _dgrad(o['dy'], w, x.shape, stride, pad) if do_dgrad else None
        dw = _wgrad(o['x_w'], o['dy_w'], wshape, stride, pad, None if dw0 is None else dw0.clone())
        return y, dx, dw
    (y, dx, dw), seen = _instances(run)
    claim = [CONV(g['n_tile'], False), WGRAD(wg['n_tile'])] + ([CONV(min(cin, 128), True)] if do_dgrad else [])
    _claim(seen, claim, f'conv {name} {"exact" if exact else "random"}')

    pre, A, n_red = B.dense_conv_ref(x, w, stride, pad, o['bias'], o['res'])
    ref = pre.clamp(min=0)
    if exact:
        B.assert_exact(y, ref, A, f'{name} fwd')
    else:
        r = B.assert_within(y, ref, A, n_red, B.OUT_REL_BF16, f'{name} fwd')
        B.assert_rejects(B.conv_fwd_faults(y, pre, x, w, stride, pad, True, g['tile']), ref, A, n_red, B.OUT_REL_BF16)
    if do_dgrad:
        ref_dx, A, n_red = B.dense_dgrad_ref(o['dy'], w, x.shape, stride, pad)
        if exact:
            B.assert_exact(dx, ref_dx, A, f'{name} dgrad')
        else:
            r = max(r, B.assert_within(dx, ref_dx, A, n_red, B.OUT_REL_BF16, f'{name} dgrad'))
            tile = B.conv_tma_geometry(*_pixels(dims, S, n), cin, sms)['tile']
            B.assert_rejects(B.conv_dgrad_faults(dx, ref_dx, o['dy'], w, x.shape, stride, pad, tile), ref_dx, A, n_red,
                             B.OUT_REL_BF16)
    ref_dw, A, n_red = B.dense_wgrad_ref(o['x_w'], o['dy_w'], wshape, stride, pad)
    if exact:
        B.assert_exact(dw, ref_dw, A, f'{name} wgrad', out_bf16=False)
        # on random operands one split's partial grows like sqrt(pixels) while the bound grows like pixels: the bound
        # sees a dropped split on the integer operands, where the partial is a non-zero integer
        if wg['n_splits'] >= 2:
            B.assert_rejects(B.wgrad_split_faults(dw, o['x_w'], o['dy_w'], wshape, stride, pad, wg), ref_dw, A, n_red,
                             B.OUT_REL_F32)
    else:
        r = max(r, B.assert_within(dw, dw0.double() + ref_dw, dw0.double().abs() + A, n_red + 1, B.OUT_REL_F32,
                                   f'{name} wgrad into dw0'))
        print(f'{name}: tile {g["tile"]} x {g["n_work"]} work on {g["grid"]} CTAs, wgrad box {wg["box"]} '
              f'{wg["n_splits"]} splits of {wg["tiles_per_cta"]} tiles, ratio {r:.4g}')


# wgrad cases whose split order is checked bit for bit
WGRAD_SPLIT_CASES = ['n16_3x3_res', 'n32_3x3_s2', 'n64_tn', 'n128_c1024', '3d_s2']


@pytest.mark.parametrize('name', WGRAD_SPLIT_CASES)
def test_conv_tma_wgrad_split_order(name):
    """conv_tma_wgrad_kernel writes one partial of dW per pixel-tile split and the fixed-order finish adds them in split
    order. With dy zeroed outside the pixel tiles of split s (the mirrored split rule), a call yields exactly that split's
    partial; the full call must equal dw0 + p0 + p1 + ... added in fp32 in split order. The scratch pool is first
    poisoned with a NaN call of the same size, so a partial row no CTA writes shows up as NaN."""
    dims, cin, cout, k, stride, pad, S, res, _ = CONV_CASES[name]
    sms = _sms()
    gen = torch.Generator().manual_seed(7 + sum(map(ord, name)))
    o = _operands(name, False, gen)
    n, x, dy = o['n'], o['x'], o['dy']
    wshape = (cout, cin) + (k, ) * dims
    So = _out_size(S, k, stride, pad)
    wg = B.wgrad_tma_geometry(*_pixels(dims, So, n), cin, cout, k ** dims, sms)
    assert wg['n_splits'] >= 2
    assert wg['last_split'] < wg['tiles_per_cta'], 'the last split must be shorter than the others'
    if name == 'n16_3x3_res':
        assert wg['last_slice_atoms'] < wg['per_slice'], 'the last (tap, channel) slice must be partial'
    if name == 'n64_tn':
        assert wg['box'][3] > 1, 'the pixel box must hold several whole images'
    _wgrad(torch.full_like(x, NAN), dy, wshape, stride, pad)
    dw0 = torch.randn(wshape, generator=gen).to(DEV)
    full = _wgrad(x, dy, wshape, stride, pad, dw0.clone())
    assert not bool(torch.isnan(full).any())
    split = B.tile_index(*B._px(dy).shape[:4], wg['box'], DEV) // wg['tiles_per_cta']
    assert int(split.max()) + 1 == wg['n_splits']
    acc = dw0.clone()
    for s in range(wg['n_splits']):
        keep = (split == s).to(dy.dtype)
        dys = dy * (keep if dims == 3 else keep[:, 0]).unsqueeze(1)
        acc += _wgrad(x, dys, wshape, stride, pad)
    assert torch.equal(full, acc), 'the split partials are not added onto dw in split order'


# ------------------------------------------------------------------------------------------------ non-tensor-map bodies
def _small_operands(xs, ws, exact, gen, n_red, dtype=BF):
    """Random operands, or operands in {-1, 0, 1} (integer bias) with partial sums around 16."""
    if exact:
        d = min(0.5, (16.0 / n_red) ** 0.5)
        return (B.ternary(xs, d, gen).to(DEV, dtype), B.ternary(ws, d, gen).to(DEV, dtype),
                torch.randint(-4, 5, (ws[0], ), generator=gen).float().to(DEV))
    return (torch.randn(xs, generator=gen).to(DEV, dtype), (torch.randn(ws, generator=gen) / n_red ** 0.5).to(DEV, dtype),
            torch.randn(ws[0], generator=gen).to(DEV))


@pytest.mark.parametrize('exact', [False, True], ids=['random', 'exact'])
@pytest.mark.parametrize('n,hw', [(2, (48, 64)), (3, (62, 90)), (1, (480, 640))])
def test_stem7x7(n, hw, exact):
    """stem7x7_tc_kernel (7x7 / 2 / 3 on the 3-channel image, 16 outputs, bias + ReLU): whole tiles (48x64), partial
    tiles on both axes (62x90 -> 31x45) and a full view."""
    from embodiedscan_b200._ffi import call, ptr, stream
    gen = torch.Generator().manual_seed(n * 7 + hw[0] + exact)
    x, w, b = _small_operands((n, 3, *hw), (16, 3, 7, 7), exact, gen, 147)
    Ho, Wo = _out_size(hw, 7, 2, 3)
    y = _nan((n, Ho, Wo, 16))
    xc, wc = _cl(x), _cl(w)           # held until the launch: a freed temporary's memory would be reused at once
    _, seen = _instances(lambda: call('esb_stem7x7_tc', ptr(xc), ptr(wc), ptr(b), ptr(y), n, *hw, 1, stream()))
    _claim(seen, [STEM], f'stem {n}x{hw} {exact}')
    pre, A, n_red = B.dense_conv_ref(x, w, 2, 3, b)
    y = y.movedim(-1, 1)
    if exact:
        B.assert_exact(y, pre.clamp(min=0), A, 'stem')
        return
    r = B.assert_within(y, pre.clamp(min=0), A, n_red, B.OUT_REL_BF16, 'stem')
    B.assert_rejects(B.conv_fwd_faults(y, pre, x, w, 2, 3, True, (16, 8, 1, 1)), pre.clamp(min=0), A, n_red,
                     B.OUT_REL_BF16)
    print(f'ratio {r:.4g}')


def _direct_fwd(x, w, b, res, stride, pad, relu):
    """esb_conv2d_direct_fwd: x (N, Cin, H, W), w (Cout, Cin, k, k) -> (N, Cout, Ho, Wo) written into NaN."""
    from embodiedscan_b200._ffi import call, dtype_code, ptr, stream
    n, cin, H, W = x.shape
    cout, k = w.shape[0], w.shape[2]
    y = _nan((n, *_out_size((H, W), k, stride, pad), cout), x.dtype)
    xc, wc, rc = _cl(x), _cl(w), _cl(res) if res is not None else None     # held until the launch
    call('esb_conv2d_direct_fwd', ptr(xc), ptr(wc), ptr(b), ptr(rc), ptr(y), n, H, W, cin, cout, k, k, stride, pad,
         int(relu), dtype_code(x.dtype), stream())
    return y.movedim(-1, 1)


def _direct_dgrad(dy, w, x_shape, stride, pad):
    from embodiedscan_b200._ffi import call, dtype_code, ptr, stream
    n, cin, H, W = x_shape
    cout, k = w.shape[0], w.shape[2]
    dx = _nan((n, H, W, cin), dy.dtype)
    dyc, wc = _cl(dy), _cl(w)
    call('esb_conv2d_direct_dgrad', ptr(dyc), ptr(wc), ptr(dx), n, H, W, cin, cout, k, k, stride, pad,
         dtype_code(dy.dtype), stream())
    return dx.movedim(-1, 1)


def _direct_wgrad(x, dy, w_shape, stride, pad):
    """esb_conv2d_direct_wgrad into zeros (its pixel slices add with atomics onto a zeroed dw): (Cout, Cin, k, k) fp32."""
    from embodiedscan_b200._ffi import call, dtype_code, ptr, stream
    n, cin, H, W = x.shape
    cout, k = w_shape[0], w_shape[2]
    dw = torch.zeros((cout, k, k, cin), device=DEV)
    xc, dyc = _cl(x), _cl(dy)
    call('esb_conv2d_direct_wgrad', ptr(xc), ptr(dyc), ptr(dw), n, H, W, cin, cout, k, k, stride, pad, dtype_code(x.dtype),
         stream())
    return dw.permute(0, 3, 1, 2)


@pytest.mark.parametrize('exact', [False, True], ids=['random', 'exact'])
@pytest.mark.parametrize('dtype', [BF, F32], ids=['bf16', 'fp32'])
def test_direct_fwd_c3_stem(dtype, exact):
    """conv2d_direct_fwd_kernel<bf16> and <float>: C3's 3 -> 64 7x7 / 2 stem (base_channels 64 is neither the stem kernel's
    width nor TMA-sized, so backbones._ConvBlock2D sends it here; in fp32 every convolution comes here), with bias and
    ReLU, into a NaN-filled output."""
    gen = torch.Generator().manual_seed(64 + exact)
    n, hw = 2, (62, 90)
    x, w, b = _small_operands((n, 3, *hw), (64, 3, 7, 7), exact, gen, 147, dtype)
    y, seen = _instances(lambda: _direct_fwd(x, w, b, None, 2, 3, True))
    _claim(seen, [DIRECT_FWD if dtype == BF else DIRECT_FWD_F32], f'direct fwd C3 stem {exact}' + ('' if dtype == BF else ' fp32'))
    pre, A, n_red = B.dense_conv_ref(x, w, 2, 3, b)
    if exact:
        B.assert_exact(y, pre.clamp(min=0), A, 'direct fwd', out_bf16=dtype == BF)
        return
    r = B.assert_within(y, pre.clamp(min=0), A, n_red, _out_rel(dtype), 'direct fwd')
    B.assert_rejects(B.conv_fwd_faults(y, pre, x, w, 2, 3, True, (1, 1, 1, 1)), pre.clamp(min=0), A, n_red, _out_rel(dtype))
    print(f'ratio {r:.4g}')


@pytest.mark.parametrize('exact', [False, True], ids=['random', 'exact'])
@pytest.mark.parametrize('dtype', [BF, F32], ids=['bf16', 'fp32'])
def test_direct_dgrad_stride3(dtype, exact):
    """conv2d_direct_dgrad_kernel<bf16> and <float>: the input gradient of a stride-3 convolution with TMA-sized channels
    (the TMA dgrad takes strides 1 and 2 only; in fp32 every dgrad comes here), into a NaN-filled output."""
    cin, cout, k, stride, pad, hw, n = 64, 64, 3, 3, 1, (31, 41), 2
    gen = torch.Generator().manual_seed(3 + exact)
    dy, w, _ = _small_operands((n, cout, *_out_size(hw, k, stride, pad)), (cout, cin, k, k), exact, gen, k * k * cout, dtype)
    dx, seen = _instances(lambda: _direct_dgrad(dy, w, (n, cin, *hw), stride, pad))
    _claim(seen, [DIRECT_DGRAD if dtype == BF else DIRECT_DGRAD_F32],
           f'direct dgrad stride 3 {exact}' + ('' if dtype == BF else ' fp32'))
    ref, A, n_red = B.dense_dgrad_ref(dy, w, (n, cin, *hw), stride, pad)
    if exact:
        B.assert_exact(dx, ref, A, 'direct dgrad', out_bf16=dtype == BF)
        return
    r = B.assert_within(dx, ref, A, n_red, _out_rel(dtype), 'direct dgrad')
    B.assert_rejects(B.conv_dgrad_faults(dx, ref, dy, w, (n, cin, *hw), stride, pad, (1, 1, 1, 1)), ref, A, n_red,
                     _out_rel(dtype))
    print(f'ratio {r:.4g}')


# fp32 direct convolutions at the backbone's own shapes (ResNet-18 / base 16 of C1: widths 16..128), (cin, cout, k, stride,
# pad, (H, W), images, residual). Forward: cin 24 puts the 64-element filter chunks across tap boundaries (216 = 3 x 64 + 24)
# and cout 40 is not a multiple of the 16 output channels of a thread; the 128-pixel blocks end partial.
DIRECT_FWD_CASES = {
    '3x3_s1_c24_c40_res': (24, 40, 3, 1, 1, (31, 45), 2, True),
    '3x3_s2_odd': (16, 32, 3, 2, 1, (33, 47), 2, False),
    '1x1_s2_ds': (64, 128, 1, 2, 0, (31, 45), 2, False),
    '3x3_s1_c128_res': (128, 128, 3, 1, 1, (15, 21), 3, True),
}


@pytest.mark.parametrize('exact', [False, True], ids=['random', 'exact'])
@pytest.mark.parametrize('name', list(DIRECT_FWD_CASES))
def test_direct_fwd_f32(name, exact):
    """conv2d_direct_fwd_kernel<float> with bias (+ residual) + ReLU as _ConvBlock2D calls it in fp32, into NaN."""
    cin, cout, k, stride, pad, hw, n, res = DIRECT_FWD_CASES[name]
    gen = torch.Generator().manual_seed(sum(map(ord, name)) + exact)
    x, w, b = _small_operands((n, cin, *hw), (cout, cin, k, k), exact, gen, k * k * cin, F32)
    ys = (n, cout, *_out_size(hw, k, stride, pad))
    r = (torch.randint(-4, 5, ys, generator=gen).float() if exact else torch.randn(ys, generator=gen)).to(DEV) \
        if res else None
    y, seen = _instances(lambda: _direct_fwd(x, w, b, r, stride, pad, True))
    _claim(seen, [DIRECT_FWD_F32], f'direct fwd fp32 {name} {exact}')
    assert (n * ys[2] * ys[3]) % 128, 'the last 128-pixel block must be partial'
    pre, A, n_red = B.dense_conv_ref(x, w, stride, pad, b, r)
    if exact:
        B.assert_exact(y, pre.clamp(min=0), A, f'direct fwd {name}', out_bf16=False)
        return
    ratio = B.assert_within(y, pre.clamp(min=0), A, n_red, B.OUT_REL_F32, f'direct fwd {name}')
    B.assert_rejects(B.conv_fwd_faults(y, pre, x, w, stride, pad, True, (1, 1, 1, 1)), pre.clamp(min=0), A, n_red,
                     B.OUT_REL_F32)
    print(f'ratio {ratio:.4g}')


# dgrad: the reduction runs over cout in 64-channel chunks; cout 80 and 96 end on a partial chunk. (cin, cout, k, stride,
# pad, (H, W), images)
DIRECT_DGRAD_CASES = {
    '3x3_s1_c80': (32, 80, 3, 1, 1, (31, 45), 2),
    '3x3_s2_odd_c96': (16, 96, 3, 2, 1, (33, 47), 2),
    '1x1_s2_ds': (64, 128, 1, 2, 0, (31, 45), 2),
}


@pytest.mark.parametrize('exact', [False, True], ids=['random', 'exact'])
@pytest.mark.parametrize('name', list(DIRECT_DGRAD_CASES))
def test_direct_dgrad_f32(name, exact):
    """conv2d_direct_dgrad_kernel<float> (one thread per input pixel and 16 input channels), into NaN. In the 1x1 stride-2
    case only the even pixels are reached by a tap: dx at every pixel with an odd row or column must be exactly 0."""
    cin, cout, k, stride, pad, hw, n = DIRECT_DGRAD_CASES[name]
    gen = torch.Generator().manual_seed(sum(map(ord, name)) + exact)
    dy, w, _ = _small_operands((n, cout, *_out_size(hw, k, stride, pad)), (cout, cin, k, k), exact, gen, k * k * cout, F32)
    dx, seen = _instances(lambda: _direct_dgrad(dy, w, (n, cin, *hw), stride, pad))
    _claim(seen, [DIRECT_DGRAD_F32], f'direct dgrad fp32 {name} {exact}')
    if k == 1 and stride == 2:
        odd = torch.ones(hw, dtype=torch.bool, device=DEV)
        odd[0::2, 0::2] = False
        assert bool((dx[:, :, odd] == 0).all()), 'pixels no tap reaches must be exactly 0'
    ref, A, n_red = B.dense_dgrad_ref(dy, w, (n, cin, *hw), stride, pad)
    if exact:
        B.assert_exact(dx, ref, A, f'direct dgrad {name}', out_bf16=False)
        return
    r = B.assert_within(dx, ref, A, n_red, B.OUT_REL_F32, f'direct dgrad {name}')
    B.assert_rejects(B.conv_dgrad_faults(dx, ref, dy, w, (n, cin, *hw), stride, pad, (1, 1, 1, 1)), ref, A, n_red,
                     B.OUT_REL_F32)
    print(f'ratio {r:.4g}')


# wgrad: (cin, cout, k, stride, pad, (H, W), images as a function of the SM count). cin x cout 960 and 3 x 16 are not
# multiples of the 256-pair block; the 1 x 3 images leave the taps of the first and last filter rows empty (padding only)
DIRECT_WGRAD_CASES = {
    '3x3_s1_c24_c40': (24, 40, 3, 1, 1, (31, 45), lambda sms: 2),
    '3x3_s2_c32_c64': (32, 64, 3, 2, 1, (33, 47), lambda sms: 2),
    '1x1_s2_ds': (64, 128, 1, 2, 0, (31, 45), lambda sms: 2),
    'stem_7x7_s2': (3, 16, 7, 2, 3, (62, 90), lambda sms: 2),
    'tiny_1x3': (16, 16, 3, 1, 1, (1, 3), lambda sms: sms),
}


@pytest.mark.parametrize('exact', [False, True], ids=['random', 'exact'])
@pytest.mark.parametrize('name', list(DIRECT_WGRAD_CASES))
def test_direct_wgrad_f32(name, exact):
    """conv2d_direct_wgrad_kernel<float>: one thread per (cin, cout) pair of a tap, one CTA column per slice of output
    pixels (bf16_bounds.direct_wgrad_slices), the slices meeting in fp32 atomicAdd on a zeroed dw. The atomics make the
    order of the slice sums (and so the last bits) run-dependent: on random operands only the bound holds, with
    n_red = pixels + slices; on operands in {-1, 0, 1} every partial sum is an exact integer, so the result must equal
    float64 bit for bit whatever the order, and dropping one pixel slice must fail the bound. Taps that padding leaves
    without a pixel must be exactly 0."""
    cin, cout, k, stride, pad, hw, n_of = DIRECT_WGRAD_CASES[name]
    sms = _sms()
    n = n_of(sms)
    So = _out_size(hw, k, stride, pad)
    M = n * So[0] * So[1]
    slice_len, n_slices = B.direct_wgrad_slices(M, cin, cout, k * k, sms)
    assert n_slices > 1, (slice_len, n_slices)
    gen = torch.Generator().manual_seed(sum(map(ord, name)) + exact)
    xs, ys = (n, cin, *hw), (n, cout, *So)
    if exact:
        d = min(0.5, (16.0 / M) ** 0.5)
        x, dy = B.ternary(xs, d, gen), B.ternary(ys, d, gen)
    else:
        x, dy = torch.randn(xs, generator=gen), torch.randn(ys, generator=gen)
    x, dy = x.to(DEV), dy.to(DEV)
    wshape = (cout, cin, k, k)
    dw, seen = _instances(lambda: _direct_wgrad(x, dy, wshape, stride, pad))
    _claim(seen, [DIRECT_WGRAD_F32], f'direct wgrad fp32 {name} {exact}')
    ref, A, n_red = B.dense_wgrad_ref(x, dy, wshape, stride, pad)
    empty = A.sum((0, 1)) == 0
    if name == 'tiny_1x3':
        assert bool(empty[0].all() and empty[2].all()), 'the first and last filter rows must see padding only'
    assert bool((dw[:, :, empty] == 0).all()), 'a tap without pixels must be exactly 0'
    if exact:
        B.assert_exact(dw, ref, A, f'direct wgrad {name}', out_bf16=False)
        B.assert_rejects(B.direct_wgrad_slice_faults(dw, x, dy, wshape, stride, pad, slice_len), ref, A, n_red + n_slices,
                         B.OUT_REL_F32)
        return
    r = B.assert_within(dw, ref, A, n_red + n_slices, B.OUT_REL_F32, f'direct wgrad {name}')
    print(f'{n_slices} slices of {slice_len} pixels, ratio {r:.4g}')


def test_stride3_block_dispatch():
    """A bf16 convolution with TMA-sized channels and stride 3 through backbones._ConvBlock2D, forward and backward: the
    module-level dispatch sends the forward and wgrad to the TMA kernels and the dgrad to conv2d_direct_dgrad_kernel."""
    from embodiedscan_b200.backbones import _ConvBlock2D
    cin, cout, k, stride, pad, hw, n = 64, 64, 3, 3, 1, (31, 41), 2
    gen = torch.Generator().manual_seed(3)
    x = torch.randn(n, cin, *hw, generator=gen).to(DEV, BF)
    w = (torch.randn(cout, cin, k, k, generator=gen) / (cin * k * k) ** 0.5).to(DEV, BF)
    b = torch.randn(cout, generator=gen).to(DEV)
    dy = torch.randn(n, cout, *_out_size(hw, k, stride, pad), generator=gen).to(DEV, BF)
    xd = x.contiguous(memory_format=torch.channels_last).requires_grad_(True)
    wd = w.contiguous(memory_format=torch.channels_last).requires_grad_(True)

    def run():
        y = _ConvBlock2D.apply(xd, wd, b, None, False, stride, pad)
        y.backward(dy.contiguous(memory_format=torch.channels_last))
        return y
    y, seen = _instances(run)
    _claim(seen, [CONV(64, False), DIRECT_DGRAD, WGRAD(64)], 'stride-3 block')
    pre, A, n_red = B.dense_conv_ref(x, w, stride, pad, b)
    r = B.assert_within(y, pre, A, n_red, B.OUT_REL_BF16, 'stride-3 fwd')
    ref, A, n_red = B.dense_dgrad_ref(dy, w, x.shape, stride, pad)
    r = max(r, B.assert_within(xd.grad, ref, A, n_red, B.OUT_REL_BF16, 'stride-3 dgrad'))
    ref, A, n_red = B.dense_wgrad_ref(x, dy, w.shape, stride, pad)
    # the block returns dW in bf16: one more rounding
    r = max(r, B.assert_within(wd.grad, ref, A, n_red, B.OUT_REL_BF16, 'stride-3 wgrad'))
    print(f'ratio {r:.4g}')


@pytest.mark.parametrize('C', [64, 16, 12])
@pytest.mark.parametrize('dtype', [BF, F32], ids=['bf16', 'fp32'])
def test_maxpool2d_bit_equal(dtype, C):
    """maxpool2d_nhwc_kernel<bf16, 8> (C a multiple of 8), <bf16, 1> and <float, 1> (every fp32 C): the stem's 3x3 / 2 / 1
    pooling into a NaN-filled output, bit-equal to F.max_pool2d, on an odd extent and values with many ties."""
    from embodiedscan_b200._ffi import call, dtype_code, ptr, stream
    gen = torch.Generator().manual_seed(C)
    x = torch.randint(-3, 4, (3, C, 31, 45), generator=gen).to(DEV, dtype) * 0.5
    y = _nan((3, *_out_size((31, 45), 3, 2, 1), C), dtype)
    xc = _cl(x)
    _, seen = _instances(lambda: call('esb_maxpool2d_nhwc', ptr(xc), ptr(y), 3, 31, 45, C, 3, 2, 1, dtype_code(dtype),
                                      stream()))
    _claim(seen, [POOL[8 if C % 8 == 0 else 1] if dtype == BF else POOL_F32],
           f'maxpool C {C}' + ('' if dtype == BF else ' fp32'))
    assert torch.equal(y.movedim(-1, 1), F.max_pool2d(x, 3, 2, 1))


# ------------------------------------------------------------------------------------------------ occupancy wrappers
# (cin, cout, k, stride, pad, (D, H, W), n): a Conv3d of the neck and the k2 / s2 ConvTranspose3d of its up blocks
CONV3D_MODULE_CASES = {'conv_s2': (64, 128, 3, 2, 1, (6, 10, 8), 2), 'transpose_k2': (128, 64, 2, 2, 0, (3, 5, 4), 2)}


@pytest.mark.parametrize('name', list(CONV3D_MODULE_CASES))
def test_occupancy_conv3d_module(name):
    """occupancy._conv3d in bf16 as the neck calls it, forward and backward, against float64 autograd: the layouts of
    _Conv3dTMA (OD HW I filter, the (k^3 Cin, Cout) weight gradient read back as (Cout, Cin, k, k, k)), and the k2 / s2
    transpose as a tensor-core rows GEMM with the 2x2x2 children interleaved into the fine grid."""
    import torch.nn as nn
    from embodiedscan_b200.occupancy import _conv3d
    cin, cout, k, stride, pad, dhw, n = CONV3D_MODULE_CASES[name]
    transpose = name.startswith('transpose')
    gen = torch.Generator().manual_seed(cin + cout + k)
    conv = nn.ConvTranspose3d(cin, cout, 2, 2, bias=False) if transpose else nn.Conv3d(cin, cout, k, stride, pad, bias=False)
    with torch.no_grad():
        conv.weight.copy_((torch.randn(conv.weight.shape, generator=gen) / (cin * k ** 3) ** 0.5).bfloat16().float())
    conv = conv.to(DEV)
    x = torch.randn(n, cin, *dhw, generator=gen).to(DEV, BF)
    xd = x.contiguous(memory_format=torch.channels_last_3d).requires_grad_(True)

    def run():
        y = _conv3d(conv, xd)
        y.backward(dy)
        return y
    if transpose:
        dy = torch.randn(n, cout, *(2 * s for s in dhw), generator=gen).to(DEV, BF)
        op = lambda a, b: F.conv_transpose3d(a, b, None, 2)  # noqa: E731
        n_red = dict(y=cin, dx=8 * cout, dw=x[:, 0].numel())
    else:
        dy = torch.randn(n, cout, *_out_size(dhw, k, stride, pad), generator=gen).to(DEV, BF)
        op = lambda a, b: F.conv3d(a, b, None, stride, pad)  # noqa: E731
        n_red = dict(y=cin * k ** 3, dx=cout * k ** 3, dw=dy[:, 0].numel())
    y, seen = _instances(run)
    if not transpose:
        _claim(seen, [CONV(128, False), CONV(64, True), WGRAD(128)], f'occupancy conv3d {name}')
    ref = B.bilinear_ref(op, x, conv.weight.detach().to(BF), dy)
    r = 0.0
    for nm, out in (('y', y), ('dx', xd.grad), ('dw', conv.weight.grad)):
        val, A = ref[nm]
        assert out.shape == val.shape, (nm, out.shape, val.shape)
        r = max(r, B.assert_within(out, val, A, n_red[nm], B.OUT_REL_BF16, f'{name} {nm}'))
    sw = y.detach().clone()
    sw[:, [0, 1]] = sw[:, [1, 0]]
    B.assert_rejects([('output channels 0 and 1 swapped', sw)], ref['y'][0], ref['y'][1], n_red['y'], B.OUT_REL_BF16)
    print(f'ratio {r:.4g}')


# ------------------------------------------------------------------------------------------------ point painting
def _paint_case(C, path, gen, dtype=BF):
    """Two scans of 37 views (more than one warp of views) on a 30 x 40 feature map; every view a translation by an odd
    multiple of 1/8 (so no point lies on a pixel boundary), about a fifth of them behind the camera; points on a
    quarter grid reaching past every border, so the sum and the divisor differ (bf16_bounds.paint_ref)."""
    import struct
    Bn, V, Hf, Wf, N = 2, 37, 30, 40, 1500
    tx = torch.randint(-6, 7, (Bn, V), generator=gen).double() + 0.125
    ty = torch.randint(-6, 7, (Bn, V), generator=gen).double() - 0.375
    front = torch.rand(Bn, V, generator=gen) > 0.2
    proj = torch.zeros(Bn, V, 4, 4)
    proj[..., 0, 0], proj[..., 1, 1], proj[..., 3, 3] = 1, 1, 1
    proj[..., 0, 3], proj[..., 1, 3] = tx.float(), ty.float()
    proj[..., 2, 3] = front.float() * 2 - 1                 # Z = 1 in front of the camera, -1 behind it
    meta = struct.pack('<5fii', 1.0, 1.0, 0.0, 0.0, float(Wf), 0, 0) + struct.pack('<8i', *[0] * 8) + \
        struct.pack('<72f', *[0.0] * 72)
    metas = torch.frombuffer(bytearray(meta * Bn), dtype=torch.uint8).clone()
    batch = torch.randint(0, Bn, (N, ), generator=gen).to(torch.int32)
    cxyz = torch.stack([torch.randint(-40, 4 * (Wf + 10), (N, ), generator=gen),
                        torch.randint(-40, 4 * (Hf + 10), (N, ), generator=gen),
                        torch.randint(0, 8, (N, ), generator=gen)], 1)
    pts = cxyz.double() * 0.25
    feat = torch.randn(Bn * V, Hf, Wf, C, generator=gen).to(DEV, dtype)
    dout = torch.randn(N, C, generator=gen).to(DEV, dtype)
    coords = torch.cat([batch[:, None], cxyz.to(torch.int32)], 1).contiguous().to(DEV) if path == 'coords' else None
    fpts = pts.float().contiguous().to(DEV) if path == 'fpts' else None
    return dict(Bn=Bn, V=V, Hf=Hf, Wf=Wf, N=N, tx=tx.to(DEV), ty=ty.to(DEV), front=front.to(DEV), proj=proj.to(DEV),
                metas=metas.to(DEV), batch=batch.to(DEV), pts=pts.to(DEV), feat=feat, dout=dout, coords=coords, fpts=fpts)


@pytest.mark.parametrize('path', ['coords', 'fpts'])
@pytest.mark.parametrize('C', [64, 300])
@pytest.mark.parametrize('dtype', [BF, F32], ids=['bf16', 'fp32'])
def test_paint(dtype, C, path):
    """paint_fwd_kernel and paint_bwd_pairs / paint_bwd_sum_kernel, bf16 and fp32 features (nearest-pixel painting of voxel
    rows (coords, the detector) or explicit fp32 points (fpts, the occupancy prior), C up to 512 in 16 slices per lane)
    against float64 painting: the forward into a NaN-filled output, its per-point count of valid views exactly, the
    backward into zeros and added onto a non-zero gradient (esb_paint_bwd documents +=). Both dtypes keep C_PAINT."""
    from embodiedscan_b200._ffi import call, dtype_code, ptr, stream
    gen = torch.Generator().manual_seed(C + len(path))
    c = _paint_case(C, path, gen, dtype)
    N, V, Hf, Wf = c['N'], c['V'], c['Hf'], c['Wf']
    pad_h, pad_w = float(Hf - 1), float(Wf - 1)
    fb = c['batch'] if path == 'fpts' else None
    out = _nan((N, C), dtype)
    cnt = torch.full((N, ), -1, dtype=torch.int32, device=DEV)
    dfeat = torch.zeros((c['Bn'] * V, Hf, Wf, C), device=DEV)
    dw0 = torch.randn(dfeat.shape, generator=gen).to(DEV)
    acc = dw0.clone()
    args = (ptr(c['coords']), ptr(c['fpts']), ptr(fb), N, 0.25 if path == 'coords' else 1.0, ptr(c['metas']), ptr(c['proj']), V)

    def fwd():
        call('esb_paint_fwd', *args, ptr(c['feat']), Hf, Wf, C, pad_h, pad_w, ptr(out), ptr(cnt), dtype_code(dtype),
             stream())

    def bwd():
        for d in (dfeat, acc):
            call('esb_paint_bwd', *args, ptr(c['dout']), Hf, Wf, C, pad_h, pad_w, ptr(d), dtype_code(dtype), stream())
    # two sessions: a session whose only kernel the profiler missed records nothing and is run again (_instances), which
    # only the forward (it overwrites its output) may be
    seen = _instances(fwd)[1] | _instances(bwd)[1]
    _claim(seen, PAINT if dtype == BF else PAINT_F32, f'paint C {C} {path}' + ('' if dtype == BF else ' fp32'))
    ref = B.paint_ref(c['feat'], c['pts'], c['batch'], c['tx'], c['ty'], c['front'], (pad_h, pad_w), c['dout'])
    hit, valid = ref['hit'], ref['valid']
    assert bool((hit & ~valid).any()) and bool((hit.sum(1) == 0).any()) and int(hit.sum(1).max()) > 1
    assert torch.equal(cnt.long(), valid.sum(1)), 'valid-view counts differ'
    val, A, n_red = ref['fwd']
    r = B.assert_within(out, val, A, n_red, _out_rel(dtype), 'paint fwd', c=B.C_PAINT)
    dval, dA, dn = ref['bwd']
    flat = lambda t: t.reshape(-1, C)  # noqa: E731
    r = max(r, B.assert_within(flat(dfeat), dval, dA, dn, B.OUT_REL_F32, 'paint bwd', c=B.C_PAINT))
    r = max(r, B.assert_within(flat(acc), flat(dw0).double() + dval, flat(dw0).double().abs() + dA, dn + 1, B.OUT_REL_F32,
                               'paint bwd onto a non-zero gradient', c=B.C_PAINT))
    fwd_f, bwd_f = B.paint_faults(out, flat(dfeat), ref, c['feat'], c['dout'])
    B.assert_rejects(fwd_f, val, A, n_red, _out_rel(dtype), c=B.C_PAINT)
    B.assert_rejects(bwd_f, dval, dA, dn, B.OUT_REL_F32, c=B.C_PAINT)
    print(f'ratio {r:.4g}')


# ------------------------------------------------------------------------------------------------ attention
def _attn(q, k, v, pad, scale, do, dq0=None, lse=None, o=None):
    """esb_attn_fwd (unless `o` and `lse` are given) then esb_attn_bwd; o / lse / dk / dv pre-filled with NaN."""
    from embodiedscan_b200._ffi import call, ptr, stream
    Bn, H, Lq, D = q.shape
    Lk = k.shape[2]
    p8 = pad.to(torch.uint8).contiguous() if pad is not None else None
    if o is None:
        o, lse = _nan(q.shape), _nan((Bn, H, Lq), torch.float32)
        call('esb_attn_fwd', ptr(q), ptr(k), ptr(v), ptr(p8), ptr(o), ptr(lse), Bn, H, Lq, Lk, scale, stream())
    dq = torch.zeros(q.shape, device=DEV) if dq0 is None else dq0
    dk, dv = _nan(k.shape), _nan(v.shape)
    delta = _nan((Bn, H, Lq), torch.float32)
    call('esb_attn_bwd', ptr(q), ptr(k), ptr(v), ptr(p8), ptr(o), ptr(do), ptr(lse), ptr(delta), ptr(dq), ptr(dk),
         ptr(dv), Bn, H, Lq, Lk, scale, stream())
    return o, lse, dq, dk, dv


def _attn_operands(Bn, H, Lq, Lk, kind, gen):
    q, k, v, do = (torch.randn(Bn, H, L, 32, generator=gen) for L in (Lq, Lk, Lk, Lq))
    pad = None
    if kind == 'masked':
        lens = torch.randint(max(Lk // 3, 1), Lk + 1, (Bn, ), generator=gen)
        pad = torch.arange(Lk)[None, :] >= lens[:, None]
    elif kind == 'leak':
        # the rows a partial tile of the previous head reads (tensor maps run over B*H*L rows) hold large values: the
        # keys among them are padded, the queries are live but a partial query tile of the previous head must skip them
        nk, nq = 128 - Lk % 128, 128 - Lq % 128
        # padded in even scans, live in odd ones: without the kj < Lk guard a partial key tile of scan b would also read
        # the padding flags of scan b + 1 (key_pad is indexed b * Lk + kj), and would find these rows live there
        pad = torch.zeros(Bn, Lk, dtype=torch.bool)
        pad[0::2, :nk] = True
        pad[-1] = True                                      # the last scan: every key padded
        k[:, :, :nk] *= 16
        v[:, :, :nk] = 1000.0
        q[:, :, :nq] *= 4
        do[:, :, :nq] *= 64
    if kind == 'zero_q':
        q.zero_()
        lens = torch.randint(1, Lk + 1, (Bn, ), generator=gen)
        pad = torch.arange(Lk)[None, :] >= lens[:, None]
    return [t.to(DEV, BF) for t in (q, k, v, do)] + [pad.to(DEV) if pad is not None else None]


# B, H, Lq, Lk, operands
ATTN_CASES = {
    'tiles_1': (1, 1, 128, 128, 'plain'), 'self_256': (2, 8, 256, 256, 'plain'), 'pad_300': (2, 8, 256, 300, 'masked'),
    'pad_1000': (3, 8, 256, 1000, 'masked'), 'keys_3500': (1, 8, 200, 3500, 'masked'), 'ragged_77x19': (2, 2, 77, 19, 'masked'),
    'leak_300': (3, 4, 300, 300, 'leak'), 'leak_200x90': (3, 3, 200, 90, 'leak'),
}


@pytest.mark.parametrize('name', list(ATTN_CASES))
def test_attention(name):
    """attn_fwd_kernel, attn_delta_kernel and attn_bwd_kernel per element against float64 softmax attention, with the
    bf16 intermediates (P, the stored O read by the delta kernel, dS^T) as exact terms of the bound (bf16_bounds.attn_ref).
    Lq / Lk multiples of 128 and not, Lk < 128, 3.5k keys; 'leak' cases put large values in the rows a partial tile of the
    previous head reads and pad every key of the last scan (its O, dQ, dK, dV must be exactly 0 and its lse -inf)."""
    Bn, H, Lq, Lk, kind = ATTN_CASES[name]
    gen = torch.Generator().manual_seed(Bn * 1000 + Lq + Lk)
    q, k, v, do, pad = _attn_operands(Bn, H, Lq, Lk, kind, gen)
    scale = 32 ** -0.5
    (o, lse, dq, dk, dv), seen = _instances(lambda: _attn(q, k, v, pad, scale, do))
    _claim(seen, ATTN, f'attention {name}')
    ref = B.attn_ref(q, k, v, pad, scale, do)
    r = 0.0
    for nm, out in (('o', o), ('dq', dq), ('dk', dk), ('dv', dv)):
        val, A, fixed = ref[nm]
        out_rel = B.OUT_REL_F32 if nm == 'dq' else B.OUT_REL_BF16
        r = max(r, B.assert_within(out, val, A, 1, out_rel, f'attention {nm}', fixed=fixed))
    fin = torch.isfinite(ref['lse'])
    assert torch.equal(torch.isfinite(lse), fin) and bool((lse[~fin] == -float('inf')).all())
    r = max(r, B.assert_within(lse[fin], ref['lse'][fin], B.lse_bound(ref)[fin], 1, B.OUT_REL_F32, 'attention lse'))
    if kind == 'leak':
        assert bool((o[-1] == 0).all() and (dq[-1] == 0).all() and (dk[-1] == 0).all() and (dv[-1] == 0).all())
    if kind == 'leak':
        val, A, fixed = ref['o']
        B.assert_rejects(B.attn_fwd_faults(o, q, k, v, pad, scale), val, A, 1, B.OUT_REL_BF16, fixed)
    if Lk > 128:
        val, A, fixed = ref['dq']
        B.assert_rejects(B.attn_dq_faults(dq, k, ref['dS']), val, A, 1, B.OUT_REL_F32, fixed)
    print(f'ratio {r:.4g}')


def test_attention_zero_queries_average_values():
    """Closed form: with q = 0 every live key has the same score, so O is the plain mean of V over the live keys."""
    gen = torch.Generator().manual_seed(11)
    q, k, v, do, pad = _attn_operands(3, 2, 150, 700, 'zero_q', gen)
    o, lse, *_ = _attn(q, k, v, pad, 32 ** -0.5, do)
    live = (~pad).double()[:, None, :, None]
    n = live.sum(2, keepdim=True)
    mean = (v.double() * live).sum(2, keepdim=True) / n
    A = (v.double().abs() * live).sum(2, keepdim=True) / n
    B.assert_within(o, mean.expand_as(o), A.expand_as(o), n.expand_as(o), B.OUT_REL_BF16, 'mean of V')
    assert torch.allclose(lse.double(), torch.log(n[:, 0, :, 0]).view(3, 1, 1).expand_as(lse), rtol=1e-6, atol=0)


def test_attention_dq_key_tile_order():
    """dQ is one partial per 128-key tile (attn_bwd_kernel) added in key-tile order (esb_sum_partial_rows). With every key
    outside tile j padded and the full call's lse passed in, a call yields exactly tile j's partial; the full dQ must equal
    their fp32 sum in tile order. The scratch pool is first poisoned by a call on NaN inputs of the same size."""
    Bn, H, Lq, Lk = 3, 8, 256, 1000
    gen = torch.Generator().manual_seed(5)
    q, k, v, do, pad = _attn_operands(Bn, H, Lq, Lk, 'masked', gen)
    scale = 32 ** -0.5
    nan = lambda t: torch.full_like(t, NAN)  # noqa: E731
    _attn(nan(q), nan(k), nan(v), pad, scale, nan(do))
    o, lse, dq, _, _ = _attn(q, k, v, pad, scale, do)
    assert not bool(torch.isnan(dq).any())
    acc = torch.zeros_like(dq)
    idx = torch.arange(Lk, device=DEV)
    for j in range((Lk + 127) // 128):
        only = pad | ((idx // 128) != j)[None]
        acc += _attn(q, k, v, only, scale, do, lse=lse, o=o)[2]
    assert torch.equal(dq, acc), 'dQ key-tile partials not added in tile order'


# ------------------------------------------------------------------------------------------------ census
def _step(model, batch):
    data = model.data_preprocessor(dict(inputs=batch['inputs'], data_samples=batch['data_samples']), True)
    losses = model(**data, mode='loss')
    sum(losses.values()).backward()


def census_step(variant, dtype=BF):
    """(model, batch) of the census step of `variant` in training mode with compute dtype `dtype`. C3 / C4 keep the
    published channel widths (which, with the strides, decide every instance: conv_tma_run, conv_wgrad_any, _ConvBlock2D)
    on one or two scans of two small views; C1 (the fp32 parity detector) runs on the batch of test_model_gpu.py's fp32
    training cases. Shared with the whole-library census of test_head_elementwise_bf16_gpu.py."""
    import warnings
    from embodiedscan_b200 import MODELS
    from embodiedscan_b200 import synth as SY
    torch.manual_seed(0)
    if variant == 'C2':
        cfg = SY.mv_det3d_config('C2')
        batch = SY.synth_batch(7, 1, n_views=20, H=480, W=640, n_points=100000, augment=True)
    elif variant == 'C1':
        cfg = SY.mv_det3d_config('C1')
        batch = SY.synth_batch(1, 2, n_views=2, H=240, W=320, n_points=2000, augment=True)
    elif variant == 'C3':
        cfg = SY.mv_occ_config('C3')
        batch = SY.synth_batch(1, 1, n_views=2, H=240, W=320, n_points=4000)
        for ds in batch['data_samples']:
            ds.gt_occupancy = SY.synth_occupancy(ds, cfg['point_cloud_range'], cfg['n_voxels'])
    else:
        cfg = SY.mv_grounding_config('C4')
        batch = SY.synth_batch(1, 2, n_views=2, H=240, W=320, n_points=2000)
        for i, ds in enumerate(batch['data_samples']):
            SY.add_grounding_prompt(ds, 1 + 2 * i, seed=i)
    with warnings.catch_warnings():
        warnings.simplefilter('ignore')
        model = MODELS.build(dict(cfg, compute_dtype=dtype)).to(DEV).train()
    return model, batch


def _census_model(variant):
    """One bf16 training forward + backward of `variant` under the profiler (in the child)."""
    model, batch = census_step(variant)
    return _instances(lambda: _step(model, batch))[1]


@pytest.mark.parametrize('variant', ['C2', 'C3', 'C4'])
def test_step_launches_only_pinned_dense_instances(variant):
    """Every dense-branch kernel instance (conv_tma*, conv2d_direct*, stem7x7*, maxpool2d*, attn*) that one bf16 training
    step launches must be one the cases above pin: a change that routes a layer to a new instance fails here until a case
    pins it."""
    seen = _claim(_census_model(variant) if _CHILD is not None else set(), [], f'{variant} bf16 step')
    assert seen, 'the profiler saw no dense-branch kernel'
    assert seen <= PINNED, f'instances no case pins: {sorted(seen - PINNED)}'
