"""Per-element error bounds for the bf16 kernels of the training steps, their float64 references, and the faults the
bounds must catch.

A kernel output `out` (bf16 operands, fp32 accumulation) is checked element by element against a float64 reference `ref`
computed from the same bf16-rounded operands:

    |out - ref| <= out_rel * |ref| + c * 2^-24 * n_red * A

`out_rel` is one rounding of the output type (2^-8 for bf16 outputs, which carry 8 significant bits; 2^-24 for fp32 outputs)
and the second term is fp32 accumulation over `n_red` terms, `A` being the same computation on absolute values (the textbook
gamma_n bound has c = 1). Elements whose every term is zero (a tile with no neighbour, an offset with no pair) have ref = 0
and A = 0, so they must be exactly zero.

C_ACC, the `c` every check uses, is the measured worst ratio times a margin. On an H100 SXM (132 SMs) the largest ratio
(|out - ref| - out_rel |ref|)+ / (2^-24 n_red A) over every case of tests/test_sparse_bf16_gpu.py was 0.165, from the
tensor-core wgrad accumulating into a non-zero dw on offsets with few pairs (a handful of fp32 additions, each rounding at
the scale of dw); the forward / dgrad kernels stay below 0.004 and the normalisations below 0.0015. C_ACC = 0.5 leaves a
factor 3 over that and is half the textbook constant. The sensitivity self-test (`assert_rejects`) checks that at this c the
bound still rejects each fault listed in `conv_faults` / `wgrad_faults`, on the H100 output and, in the CPU suite, on a
bf16-emulated output. The normalisations use the same form with their own A and n_red (`seg_norm_ref`).

The dense branch (tests/test_dense_bf16_gpu.py) uses the same C_ACC. On an H100 SXM (80 GB HBM3, 132 SMs, 700 W power
limit) its worst ratios were: 0.0245 for the TMA convolutions (forward, dgrad and wgrad into a non-zero dw, 2-D and 3-D;
the largest from a 3-D wgrad with 768 input channels), 0.00096 for the occupancy Conv3d / ConvTranspose3d wrappers,
0.00044 for the 7x7 stem, 0.00084 for the SIMT direct kernels, and 0.337 for attention (from the cases whose key rows of
16x magnitude and values of 1000 are live in every other scan, scores up to a few hundred; 0.131 on plain random
operands; the bf16 intermediates are exact terms outside c, see `attn_ref`). The
TMA convolutions, the stem and the direct forward / dgrad also matched the float64 result bit for bit on operands in
{-1, 0, 1}: the fp32 accumulation (wgmma's included) is exact on such integers. The dense faults are `conv_fwd_faults`,
`conv_dgrad_faults`, `wgrad_split_faults` (on integer operands: on random ones a dropped split of a long pixel reduction
is below the bound's resolution), `attn_fwd_faults`, `attn_dq_faults` and `paint_faults`; the selection-rule mirrors `conv_tma_geometry` / `wgrad_tma_geometry` let each case assert the geometry it
names from the SM count.

Painting has its own constant, C_PAINT = 1.0 (the textbook one): its backward adds a handful of pairs per pixel, each
term rounded twice (1 / count and the product) before the sum, and onto a non-zero gradient the worst ratio measured on
the same H100 was 0.54, above C_ACC; its forward stays below C_ACC.

The head, loss and elementwise kernels (tests/test_head_elementwise_bf16_gpu.py) use C_ACC too. On the same H100 SXM
(700 W power limit) their worst ratios were: 0.0667 for the focal loss (sum and per-element gradient, fp32 and bf16
logits, the C2-size sum included; the conditioning K(x) = 1 + e^|x| of `focal_ref` is in the element term, not in c),
0.284 for bias_act_kernel (the fp32 cases, one rounding of x + bias; every bf16 case rounds to the reference exactly),
0.367 for act_bwd_kernel (fp32 ELU; without its `fixed` term, reading ELU's derivative from the bf16 output would need
c = 4.2e6), 0.152 for interp_features_kernel, and 0.0015 for the BatchNorm / InstanceNorm instances with ELU (their
backward carrying the same `fixed` term through the normalisation's backward, `seg_norm_bwd_fixed`). The faults are
`focal_faults_fwd`, `focal_faults_bwd`, `bias_act_faults`, `act_bwd_faults` and `interp_faults`.

The fp32 instances (the parity arithmetic; the fp32 cases of the three modules) use the same form with out_rel =
OUT_REL_F32 = 2^-24 and the same C_ACC. Where an fp32 kernel calls rsqrtf or expm1f (the normalisations, ELU), the
function's documented maximum error (ULP_RSQRTF, ULP_EXPM1F) is an explicit `fixed` term (`seg_norm_fn_fixed`), and the
ELU backward keeps its `fixed` term for reading the derivative as y + 1, with the fp32 output rounding. On an H100 SXM
(80 GB HBM3, 132 SMs, 700 W power limit) the worst fp32 ratios were: 0.067 for the SIMT sparse forward / dgrad
(spconv_fwd_kernel<float, *>, from the stem's dgrad; 0.058 at cin 33 / cout 70, 0.0045 at 640 -> 640), 0.312 for the
SIMT wgrad (640 -> 640, one split, into a non-zero dw; 0.228 with six splits), 0.0122 for the two-pass normalisations
(InstanceNorm, C = 64; the BatchNorms below 0.0015), 0.051 for the direct 2-D forward (a 1x1 stride-2 downsample), 0.026
for its dgrad, 0.0018 for its wgrad (n_red = pixels + slices: its atomics add the pixel slices in any order), and 0.55
for painting (under C_PAINT). Pooling and the image normalisation are bit-exact in fp32 too, and every fp32 convolution family is bit-exact on
operands in {-1, 0, 1}. One case needs more than C_ACC: the fp32 forward of the sparse stem (3 input channels), 0.504.
Its rows sum a few 3-term dot products, too few terms for the roundings of the partial sums to average out. An fma chain
over n terms is off by at most (n - 1) 2^-24 A beyond the output rounding, a ratio of (n - 1) / n: below 1, the textbook
constant, which that case uses (C_SHORT_F32). In bf16 the output rounding hides this (0.0034). The new faults are
`direct_wgrad_slice_faults` (a dropped pixel slice, on integer operands) and `wgrad_faults` at the SIMT split length;
`simt_wgrad_splits` and `direct_wgrad_slices` mirror the two selection rules.

Nothing here imports the library: it runs on CPU tensors as well as CUDA tensors.
"""
import math

import torch

U32 = 2.0 ** -24
OUT_REL_BF16 = 2.0 ** -8
OUT_REL_F32 = 2.0 ** -24
C_ACC = 0.5
C_PAINT = 1.0
C_SHORT_F32 = 1.0


# ------------------------------------------------------------------------------------------------ the bound
def excess_ratio(out, ref, A, n_red, out_rel, fixed=0.0):
    """The smallest c for which `out` passes: max over elements of (|out - ref| - out_rel |ref| - fixed)+ / (2^-24 n_red A).
    `fixed` is the part of the bound that is exact rather than a multiple of c (the bf16 intermediates of attention).
    inf when an element whose bound is exactly zero (ref = A = 0) is not exactly zero, or when `out` holds a NaN."""
    err = (out.double() - ref).abs()
    excess = (err - out_rel * ref.abs() - fixed).clamp(min=0)
    if torch.isnan(err).any():
        return math.inf
    scale = U32 * n_red * A
    scale = torch.broadcast_to(torch.as_tensor(scale, dtype=torch.float64, device=ref.device), excess.shape)
    if bool(((excess > 0) & (scale == 0)).any()):
        return math.inf
    r = torch.where(excess > 0, excess / torch.where(scale > 0, scale, 1.0), torch.zeros_like(excess))
    return float(r.max()) if r.numel() else 0.0


def within(out, ref, A, n_red, out_rel, c=C_ACC, fixed=0.0):
    err = (out.double() - ref).abs()
    return bool((err <= out_rel * ref.abs() + fixed + c * U32 * n_red * A).all())


def assert_within(out, ref, A, n_red, out_rel, what, fixed=0.0, c=C_ACC):
    """Assert the bound at `c` (C_ACC unless a family has its own); returns the ratio the output needed."""
    r = excess_ratio(out, ref, A, n_red, out_rel, fixed)
    assert within(out, ref, A, n_red, out_rel, c, fixed), f'{what}: needs c = {r:.3g} > {c}'
    return r


def assert_rejects(faults, ref, A, n_red, out_rel, fixed=0.0, c=C_ACC):
    """Every faulty copy of a correct output must fail the bound, else the bound is too loose to see that fault."""
    passed = [name for name, bad in faults if within(bad, ref, A, n_red, out_rel, c, fixed)]
    assert not passed, f'the bound accepts these faults: {passed}'


# ------------------------------------------------------------------------------------------------ references
def gather_gemm(x, w, nbr, w_layout=1, dtype=torch.float64):
    """y[o] = sum over offsets k with nbr[k, o] >= 0 of x[nbr[k, o]] @ W_k, one offset at a time, in `dtype`.
    w_layout 1: w is (K, cin, cout) and W_k = w[k]; w_layout 0: w is (K, cout, cin) and W_k = w[k]^T.
    Returns (y, A = the same with |x| and |w|, n_red = (used offsets of row o) * cin as an (n_out, 1) column)."""
    xs, ws = x.to(dtype), w.to(dtype)
    if w_layout == 0:
        ws = ws.transpose(1, 2)
    K, n_out = nbr.shape
    cin, cout = ws.shape[1], ws.shape[2]
    y = torch.zeros((n_out, cout), dtype=dtype, device=x.device)
    A = torch.zeros_like(y)
    cnt = torch.zeros((n_out, 1), dtype=dtype, device=x.device)
    for k in range(K):
        sel = torch.nonzero(nbr[k] >= 0).squeeze(1)
        if sel.numel() == 0:
            continue
        g = xs[nbr[k, sel].long()]
        y[sel] += g @ ws[k]           # one offset feeds each output row at most once: no duplicate indices
        A[sel] += g.abs() @ ws[k].abs()
        cnt[sel] += 1
    return y, A, cnt * cin


def pair_wgrad(x, dy, pin, pout, koff, dtype=torch.float64):
    """dW[k] = x[pin[p]]^T dy[pout[p]] summed over the pairs p of offset k (koff: K + 1 host ints), in `dtype`.
    Returns (dW (K, cin, cout), A, n_red = pairs of offset k as a (K, 1, 1) column)."""
    xs, ds = x.to(dtype), dy.to(dtype)
    K = len(koff) - 1
    g = torch.zeros((K, x.shape[1], dy.shape[1]), dtype=dtype, device=x.device)
    A = torch.zeros_like(g)
    n = torch.zeros((K, 1, 1), dtype=dtype, device=x.device)
    for k in range(K):
        b, e = koff[k], koff[k + 1]
        if e > b:
            a, d = xs[pin[b:e].long()], ds[pout[b:e].long()]
            g[k], A[k], n[k] = a.t() @ d, a.abs().t() @ d.abs(), e - b
    return g, A, n


def seg_norm_ref(x, sizes, gamma, beta, eps, res=None, pivot=False):
    """Segmented normalisation in float64: z = (x - mean_s) * rstd_s * gamma + beta (+ res) over row segments of `sizes`
    (biased variance). Returns (z before the activation, A, n_red, stats) where n_red is the row count of the element's
    segment and A bounds the magnitudes an fp32 evaluation rounds: |x - mean|, |mean| and mean|x - mean| scaled by
    rstd |gamma|, then |beta| and |res|. pivot=True models the single-pass statistics of the fused BatchNorm, which sum
    (x - x[0]) and its square: their variance loses (1 + ((x[0] - mean) rstd)^2) times more to cancellation."""
    xs = x.double()
    seg = torch.repeat_interleave(torch.arange(len(sizes), device=x.device), torch.tensor(sizes, device=x.device))
    S, C = len(sizes), x.shape[1]
    mean = torch.zeros((S, C), dtype=torch.float64, device=x.device).index_add_(0, seg, xs)
    n = torch.tensor(sizes, dtype=torch.float64, device=x.device).view(S, 1)
    mean /= n
    d = xs - mean[seg]
    var = torch.zeros_like(mean).index_add_(0, seg, d * d) / n
    rs = torch.rsqrt(var + eps)
    m1 = torch.zeros_like(mean).index_add_(0, seg, d.abs()) / n
    w = 1 + ((xs[0] - mean) * rs) ** 2 if pivot else torch.ones_like(mean)
    g, b = gamma.double().view(1, C), beta.double().view(1, C)
    z = d * rs[seg] * g + b
    A = (d.abs() + mean[seg].abs() + m1[seg]) * w[seg] * rs[seg] * g.abs() + b.abs()
    if res is not None:
        z = z + res.double()
        A = A + res.double().abs()
    return z, A, n[seg], dict(seg=seg, n=n, mean=mean, rs=rs, w=w, m=mean.abs() * rs + m1 * rs)


def seg_norm_bwd_ref(x, gy, gamma, st):
    """Backward of seg_norm_ref given gy = dy * act'(y) (the activation's derivative read from the kernel's own output):
    dx = gamma rstd (gy - mean_s(gy) - xhat mean_s(gy xhat)), dbeta = sum gy, dgamma = sum gy xhat, each with its A.
    Returns ((dx, A), (dgamma, A), (dbeta, A)); n_red is the segment's rows for dx and all rows for dgamma / dbeta."""
    seg, n, rs, w, m = st['seg'], st['n'], st['rs'], st['w'], st['m']
    S, C = n.shape[0], x.shape[1]
    xh = (x.double() - st['mean'][seg]) * rs[seg]
    g = gy.double()
    P = torch.zeros((S, C), dtype=torch.float64, device=x.device)
    sg, sgx = P.clone().index_add_(0, seg, g), P.clone().index_add_(0, seg, g * xh)
    pa, qa = P.clone().index_add_(0, seg, g.abs()) / n, P.clone().index_add_(0, seg, (g * xh).abs()) / n
    gm = gamma.double().view(1, C)
    dx = gm * rs[seg] * (g - sg[seg] / n[seg] - xh * sgx[seg] / n[seg])
    A_dx = gm.abs() * rs[seg] * w[seg] * (g.abs() + pa[seg] + (xh.abs() + m[seg]) * (qa[seg] + pa[seg] * (1 + m[seg])))
    db, A_db = sg.sum(0), (pa * n).sum(0)
    dg = sgx.sum(0)
    A_dg = (((g * xh).abs() + g.abs() * (xh.abs() + m[seg])) * w[seg]).sum(0)
    return (dx, A_dx), (dg, A_dg), (db, A_db)


# The documented maximum errors of the CUDA single-precision functions the fp32 kernels call (CUDA C++ Programming Guide,
# "Mathematical Functions", single precision), in ulps; one ulp of an fp32 value v is at most ULP |v|. They enter the fp32
# bounds as explicit `fixed` terms, not through c.
ULP = 2.0 ** -23
ULP_RSQRTF = 2
ULP_EXPM1F = 1


def seg_norm_fn_fixed(x, gamma, st, z, act, gy=None):
    """What rsqrtf and expm1f may add to an fp32 normalisation beyond the roundings c covers. rstd = rsqrtf(var + eps) is
    off by e = ULP_RSQRTF ULP relative, which moves z by e |xhat gamma|; ELU's expm1f adds ULP_EXPM1F ULP |y| where z <= 0.
    With `gy` (dy act'(y)) also the backward: dx = gamma rs (g - mean g - xhat mean(g xhat)) reads rs once and xhat twice
    (directly and through sum g xhat), so it moves by 3 e |gamma| rs (|g| + mean|g| + |xhat| mean|g xhat|); dgamma =
    sum g xhat by e sum |g xhat|; dbeta not at all. Returns F_y, or (F_y, F_dx, F_dgamma, F_dbeta)."""
    seg, n, rs = st['seg'], st['n'], st['rs']
    e = ULP_RSQRTF * ULP
    xh = ((x.double() - st['mean'][seg]) * rs[seg]).abs()
    gm = gamma.double().abs().view(1, -1)
    F_y = e * xh * gm
    if act == 2:
        F_y = F_y + ULP_EXPM1F * ULP * torch.expm1(z.clamp(max=0)).abs()
    if gy is None:
        return F_y
    g = gy.double().abs()
    S, C = n.shape[0], x.shape[1]
    P = torch.zeros((S, C), dtype=torch.float64, device=x.device)
    pa, qa = P.clone().index_add_(0, seg, g) / n, P.clone().index_add_(0, seg, g * xh) / n
    F_dx = 3 * e * gm * rs[seg] * (g + pa[seg] + xh * qa[seg])
    return F_y, F_dx, e * (g * xh).sum(0), torch.zeros(C, dtype=torch.float64, device=x.device)


# ------------------------------------------------------------------------------------------------ faults
def conv_faults(out, x, w, nbr, w_layout=1, tile_rows=128, chunk=64):
    """Copies of a correct gather-GEMM output with one fault each, as a tile kernel could make them:
    the contribution of the sparsest used kernel offset missing, output channels 0 and 1 swapped, the last `chunk`-channel
    slice of the reduction (partial when chunk does not divide cin) missing, and the last (partial) `tile_rows`-row tile
    left at zero."""
    K, n_out = nbr.shape
    assert n_out % tile_rows, 'the last row tile must be partial'
    cin = x.shape[1]
    used = [(int((nbr[k] >= 0).sum()), k) for k in range(K) if bool((nbr[k] >= 0).any())]
    k_min = min(used)[1]
    one = torch.full_like(nbr, -1)
    one[k_min] = nbr[k_min]
    drop_k = gather_gemm(x, w, one, w_layout)[0]
    c0 = (cin - 1) // chunk * chunk
    xs = x.clone()
    xs[:, :c0] = 0
    drop_slice = gather_gemm(xs, w, nbr, w_layout)[0]
    swapped = out.clone()
    swapped[:, [0, 1]] = out[:, [1, 0]]
    tail = out.clone()
    tail[n_out // tile_rows * tile_rows:] = 0
    return [(f'kernel offset {k_min} dropped', (out.double() - drop_k).to(out.dtype)),
            ('output channels 0 and 1 swapped', swapped),
            (f'reduction channels {c0}..{cin - 1} zeroed', (out.double() - drop_slice).to(out.dtype)),
            ('last partial row tile left at zero', tail)]


def wgrad_faults(out, x, dy, pin, pout, koff, chunk_pairs):
    """A correct weight gradient with its smallest pair chunk (`chunk_pairs` consecutive pairs of one offset) missing."""
    chunks = []
    for k in range(len(koff) - 1):
        for b in range(koff[k], koff[k + 1], chunk_pairs):
            chunks.append((min(b + chunk_pairs, koff[k + 1]) - b, k, b))
    n, k, b = min(chunks)
    a, d = x[pin[b:b + n].long()].double(), dy[pout[b:b + n].long()].double()
    bad = out.double().clone()
    bad[k] -= a.t() @ d
    return [(f'pair chunk of offset {k} at pair {b} ({n} pairs) dropped', bad.to(out.dtype))]


# ------------------------------------------------------------------------------------------------ selection rules
def tc_fwd_n_tile(n_out, cout, sms):
    """The N_TILE esb_spconv_tc_fwd picks (csrc/spconv_tc.cu): the widest tile that still gives every SM a CTA."""
    row_tiles = (n_out + 127) // 128
    if cout % 256 == 0 and row_tiles * (cout // 256) >= sms:
        return 256
    if cout % 128 == 0 and row_tiles * (cout // 128) >= sms:
        return 128
    return 64


def tc_wgrad_chunk_pairs(n_pairs_hint, cin, cout, sms):
    """The pair-chunk length esb_spconv_tc_wgrad picks (csrc/spconv_tc.cu)."""
    n_tile = 128 if cout % 128 == 0 else 64
    tiles = (cin + 127) // 128 * (cout // n_tile)
    target = (8 * sms + tiles - 1) // tiles
    cp = (n_pairs_hint // 2 + target - 1) // target
    cp = (cp + 63) // 64 * 64
    return min(max(cp, 512), 16384)


def simt_wgrad_splits(n_pairs_hint, K, cin, cout, sms):
    """The pair splits esb_spconv_wgrad picks (csrc/spconv.cu, spconv_wgrad): ~4 CTAs per SM over the 64 x 64 (cin, cout)
    tiles of every offset, at least 256 pairs per split on average, 1..64. Split s of an offset with n pairs holds pairs
    [s per, (s + 1) per) with per = ceil(n / splits) (`simt_wgrad_split_len`); the partials are added in split order."""
    tiles = K * _cdiv(cin, 64) * _cdiv(cout, 64)
    splits = min(4 * sms // tiles, (n_pairs_hint // K + 1) // 256 + 1)
    return min(max(splits, 1), 64)


def simt_wgrad_split_len(n_pairs, splits):
    return _cdiv(n_pairs, splits)


def direct_wgrad_slices(M, cin, cout, taps, sms):
    """(slice, n_slices) esb_conv2d_direct_wgrad picks (csrc/conv2d_direct.cu): enough (256-pair block, tap, slice) CTAs
    to give each SM ~32, at most 1024 slices, at least 64 output pixels each; slice z holds pixels [z slice, (z+1) slice)
    of the M = N Ho Wo output pixels and adds its partial to dw with fp32 atomics."""
    pair_blocks = _cdiv(cin * cout, 256)
    slices = min(4 * sms * 8 // (pair_blocks * taps) + 1, 1024)
    slice_len = max(_cdiv(M, slices), 64)
    return slice_len, _cdiv(M, slice_len)


def random_kernel_map(n_in, n_out, K, gen, device='cpu', empty_offset=None, single_offset=None, empty_tile=None,
                      tile_rows=128):
    """nbr (K, n_out) int32: through each offset an injective map into [0, n_in) of random density (as a real kernel map
    is); `empty_offset` gets no neighbour at all, `single_offset` exactly one, and the `tile_rows` rows of `empty_tile`
    none."""
    nbr = torch.full((K, n_out), -1, dtype=torch.int32)
    for k in range(K):
        dens = 0.1 + 0.5 * float(torch.rand((), generator=gen))
        keep = torch.rand(n_out, generator=gen) < dens
        src = torch.randperm(n_in, generator=gen)[:n_out].to(torch.int32)
        nbr[k] = torch.where(keep, src, -1)
    if empty_offset is not None:
        nbr[empty_offset] = -1
    if single_offset is not None:
        o = int(torch.randint(n_out, (), generator=gen))
        v = int(torch.randint(n_in, (), generator=gen))
        nbr[single_offset] = -1
        nbr[single_offset, o] = v
    if empty_tile is not None:
        nbr[:, empty_tile * tile_rows:(empty_tile + 1) * tile_rows] = -1
    return nbr.to(device)


def random_pairs(counts, n_in, n_out, gen, device='cpu'):
    """Pair lists (pin, pout int32, koff host list) with counts[k] pairs for offset k; output rows ascend within an offset
    and no output row repeats, as in the library's compacted lists."""
    pin, pout, koff = [], [], [0]
    for c in counts:
        pout.append(torch.sort(torch.randperm(n_out, generator=gen)[:c]).values)
        pin.append(torch.randperm(n_in, generator=gen)[:c])
        koff.append(koff[-1] + c)
    pin = torch.cat(pin).to(torch.int32).to(device)
    pout = torch.cat(pout).to(torch.int32).to(device)
    return pin, pout, koff


# ================================================================================================ dense branch
# The image backbone, the occupancy Conv3d neck and the grounding attention. Tensors here are in torch's layout (N, C, *S)
# and filters (Cout, Cin, *k); the tests convert to and from the kernels' channels-last memory.
def _conv_ops(dims):
    F = torch.nn.functional
    if dims == 2:
        return F.conv2d, torch.nn.grad.conv2d_input, torch.nn.grad.conv2d_weight
    return F.conv3d, torch.nn.grad.conv3d_input, torch.nn.grad.conv3d_weight


def dense_conv_ref(x, w, stride, pad, bias=None, res=None):
    """Forward of a 2-D / 3-D convolution in float64 (fp32 bias, bf16 residual): (y before the activation, A,
    n_red = taps * cin + 2). The caller applies ReLU to y (1-Lipschitz: the bound carries over)."""
    conv = _conv_ops(w.dim() - 2)[0]
    xs, ws = x.double(), w.double()
    y, A = conv(xs, ws, None, stride, pad), conv(xs.abs(), ws.abs(), None, stride, pad)
    shape = (1, -1) + (1, ) * (w.dim() - 2)
    if bias is not None:
        y, A = y + bias.double().view(shape), A + bias.double().abs().view(shape)
    if res is not None:
        y, A = y + res.double(), A + res.double().abs()
    return y, A, w[0].numel() + 2


def dense_dgrad_ref(dy, w, x_shape, stride, pad):
    """dL/dx of the convolution in float64: (dx, A, n_red = taps * cout)."""
    dgrad = _conv_ops(w.dim() - 2)[1]
    ws, ds = w.double(), dy.double()
    return (dgrad(x_shape, ws, ds, stride, pad), dgrad(x_shape, ws.abs(), ds.abs(), stride, pad),
            w.shape[0] * w[0, 0].numel())


def dense_wgrad_ref(x, dy, w_shape, stride, pad):
    """dL/dw of the convolution in float64: (dw (Cout, Cin, *k), A, n_red = N * output pixels)."""
    wgrad = _conv_ops(len(w_shape) - 2)[2]
    xs, ds = x.double(), dy.double()
    return (wgrad(xs, w_shape, ds, stride, pad), wgrad(xs.abs(), w_shape, ds.abs(), stride, pad), dy[:, 0].numel())


def ternary(shape, density, gen):
    """Exact-arithmetic operands: each element is 0, or +-1 with probability `density` (random sign)."""
    nz = torch.rand(shape, generator=gen) < density
    return torch.where(nz, torch.randint(0, 2, shape, generator=gen).float() * 2 - 1, torch.zeros(shape))


def assert_exact(out, ref, A, what, out_bf16=True):
    """On operands in {-1, 0, 1} (integer bias / residual) every product is exact and every partial sum is an integer of
    magnitude <= A; with A <= 2^11 the fp32 accumulation is exact whatever its order, and with |ref| <= 256 so is the bf16
    output. The output must then equal the float64 reference bit for bit."""
    assert float(A.max()) <= 2 ** 11, f'{what}: partial sums up to {float(A.max())} (> 2^11): lower the density'
    if out_bf16:
        assert float(ref.abs().max()) <= 256, f'{what}: |y| up to {float(ref.abs().max())} is not exact in bf16'
    bad = int((out.double() != ref).sum())
    assert bad == 0, f'{what}: {bad} of {out.numel()} elements differ from the exact result'


# ------------------------------------------------------------------------------------------------ attention
def attn_ref(q, k, v, key_pad, scale, do=None):
    """softmax(q k^T scale + key padding) v in float64 for q (B,H,Lq,D), k / v (B,H,Lk,D), key_pad (B,Lk) bool (True =
    padded) or None, and with `do` its backward. Returns {name: (value, A, fixed)} for 'o', 'dq', 'dk', 'dv' (n_red is
    folded into A: pass n_red = 1) plus 'lse' (natural log, -inf for a scan whose keys are all padded) and the
    intermediates 'P', 'dS'.

    Every bound is |out - ref| <= 2^-8 |ref| + fixed + c 2^-24 A, where `fixed` collects the bf16 intermediates that
    csrc/attn_tc.cu documents. One rounding to bf16 (8 significant bits) is off by <= u = 2^-8 of its value; `fixed`
    carries a factor (1 + 2^-7) so that the output rounding of a value already off by `fixed` stays covered:
      * O = sum_j bf16(p_j) V_j / l with l summed from the unrounded p: rounding P moves O by <= u sum_j P_ij |V_j|
        = u (P|V|)_i.  The same for dV = bf16(P)^T dO: u (P^T |dO|).
      * delta_i = sum_d bf16(O)_id dO_id (attn_delta_kernel reads the stored O): the stored O is off by its output rounding
        and the P rounding above, each <= u (P|V|)_id, so delta is off by <= E_i = 2u sum_d (P|V|)_id |dO_id|, and
        dS_ij = P_ij (dP_ij - delta_i) scale by P_ij scale E_i.
      * dS^T is stored bf16 for dK = dS^T Q and dQ = dS K: u |dS_ij|.
      So fixed(dS) = P scale E + u |dS|, fixed(dK) = fixed(dS)^T |Q|, fixed(dQ) = fixed(dS) |K|.
    The fp32 part: a score is a 32-term dot product (error <= 32 2^-24 scale |q|.|k|); p = exp2(s log2e - m) rounds the
    product, the subtraction and exp2 (a few ulps), and the lse it subtracts in the backward carries the error of l (a sum
    of n_live terms). So p_ij is off by a relative 2^-24 Z_ij, Z = 32 Sabs + 2|S| + 2(|m| + |lse|) + n_live + 8, and
      A(O)  = n_live (P|V| + |O|) + (P o Z)|V| + (P o Z)1 |O|        (O = sum p V / sum p moves by sum P eps (V - O))
      A(dV) = Lq P^T|dO| + (P o Z)^T |dO|
      C(dS) = P scale (32 |dO||V|^T + Z |dP - delta| + 32 sum_d |O||dO|) + 3 |dS|
      A(dK) = Lq |dS|^T |Q| + C(dS)^T |Q|,   A(dQ) = n_live |dS| |K| + C(dS) |K|."""
    qd, kd, vd = q.double(), k.double(), v.double()
    B, H, Lq, D = q.shape
    Lk = k.shape[2]
    live = torch.ones((B, Lk), dtype=torch.bool, device=q.device) if key_pad is None else ~key_pad.bool()
    live4 = live[:, None, None, :]
    n_live = live.sum(-1).double().view(B, 1, 1, 1)
    S = scale * qd @ kd.transpose(-1, -2)
    Sabs = scale * qd.abs() @ kd.abs().transpose(-1, -2)
    Sm = S.masked_fill(~live4, -math.inf)
    lse = torch.logsumexp(Sm, -1)
    fin = torch.isfinite(lse)[..., None]
    lse_f = torch.where(fin, lse[..., None], 0.0)
    m_f = torch.where(fin, Sm.amax(-1, keepdim=True), 0.0)
    P = torch.where(live4, torch.exp(S - lse_f), 0.0)
    Z = 32 * Sabs + 2 * S.abs() + 2 * (m_f.abs() + lse_f.abs()) + n_live + 8
    PZ = P * Z
    va = vd.abs()
    O = P @ vd
    PV = P @ va
    u = 2.0 ** -8 * (1 + 2.0 ** -7)
    out = dict(o=(O, n_live * (PV + O.abs()) + PZ @ va + PZ.sum(-1, keepdim=True) * O.abs(), u * PV),
               lse=lse, P=P)
    if do is None:
        return out
    dod = do.double()
    da = dod.abs()
    dP = dod @ vd.transpose(-1, -2)
    delta = (O * dod).sum(-1, keepdim=True)
    dS = P * (dP - delta) * scale
    E = 2 * u * (PV * da).sum(-1, keepdim=True)
    Fd = P * scale * E + u * dS.abs()
    Cd = P * scale * (32 * da @ va.transpose(-1, -2) + Z * (dP - delta).abs() + 32 * (O.abs() * da).sum(-1, keepdim=True)) \
        + 3 * dS.abs()
    Pt, dSt, Fdt, Cdt = (t.transpose(-1, -2) for t in (P, dS, Fd, Cd))
    out['dv'] = (Pt @ dod, Lq * (Pt @ da) + PZ.transpose(-1, -2) @ da, u * (Pt @ da))
    out['dk'] = (dSt @ qd, Lq * (dSt.abs() @ qd.abs()) + Cdt @ qd.abs(), Fdt @ qd.abs())
    out['dq'] = (dS @ kd, n_live * (dS.abs() @ kd.abs()) + Cd @ kd.abs(), Fd @ kd.abs())
    out['dS'] = dS
    return out


def lse_bound(ref):
    """A for the fp32 lse = (m + log2 l) ln 2 (absolute error; n_red = 1): l sums n_live terms."""
    P, lse = ref['P'], ref['lse']
    fin = torch.isfinite(lse)
    n_live = (P > 0).sum(-1).double()
    return torch.where(fin, 4 * lse.abs() + n_live + 8, 0.0)


# ------------------------------------------------------------------------------------------------ dense selection rules
def _cdiv(a, b):
    return -(-a // b)


def conv_choose_tile(Wo, Ho, Do, N):
    """choose_tile (csrc/conv_tma.cu): the output tile TW x TH x TD x TN <= 128 pixels wasting the fewest MMA rows; several
    images per tile only when one tile holds a whole image."""
    best, out = -1.0, (1, 1, 1, 1)
    for tw in range(1, min(Wo, 128) + 1):
        for th in range(1, Ho + 1):
            if tw * th > 128:
                break
            for td in range(1, Do + 1):
                if tw * th * td > 128:
                    break
                tn = min(128 // (tw * th * td), N) if (tw, th, td) == (Wo, Ho, Do) else 1
                tiles = _cdiv(Wo, tw) * _cdiv(Ho, th) * _cdiv(Do, td) * _cdiv(N, tn)
                eff = float(Wo) * Ho * Do * N / (tiles * 128.0) + 1e-6 * tw
                if eff > best:
                    best, out = eff, (tw, th, td, tn)
    return out


def conv_tma_geometry(N, Do, Ho, Wo, cout, sms):
    """What conv_tma_run launches for an output (N, Do, Ho, Wo, cout) (cout = the GEMM's N: Cin for a dgrad): N_TILE =
    min(cout, 128), the tile, the persistent grid (one CTA per SM) and the most tiles one CTA walks."""
    n_tile = min(cout, 128)
    tile = conv_choose_tile(Wo, Ho, Do, N)
    grid_t = (_cdiv(Wo, tile[0]), _cdiv(Ho, tile[1]), _cdiv(Do, tile[2]), _cdiv(N, tile[3]))
    n_work = grid_t[0] * grid_t[1] * grid_t[2] * grid_t[3] * (cout // n_tile)
    grid = min(sms, n_work)
    partial = bool(Wo % tile[0] or Ho % tile[1] or Do % tile[2] or N % tile[3])
    return dict(n_tile=n_tile, tile=tile, tiles=grid_t, n_work=n_work, grid=grid, per_cta=_cdiv(n_work, grid),
                partial=partial)


def wgrad_tma_geometry(N, Do, Ho, Wo, cin, cout, taps, sms):
    """What conv_wgrad_any / launch_wgrad_tma launch: the 64-pixel box, the (tap, channel) atoms per 128-row slice, the
    pixel-tile splits (~2 CTAs per SM over slices x channel blocks) and tiles_per_cta; the last split may be shorter."""
    best, box = -1.0, None
    p2 = [1, 2, 4, 8, 16, 32, 64]
    for tw in p2:
        for th in p2:
            for td in p2:
                if tw * th * td > 64:
                    continue
                tn = 64 // (tw * th * td)
                if tn > 1 and (tw < Wo or th < Ho or td < Do):
                    continue
                if td > 1 and Do == 1:
                    continue
                tiles = float(_cdiv(Wo, tw) * _cdiv(Ho, th) * _cdiv(Do, td) * _cdiv(N, tn))
                eff = float(Wo) * Ho * Do * N / (tiles * 64.0) + 1e-6 * tw
                if eff > best:
                    best, box = eff, (tw, th, td, tn)
    grid_t = (_cdiv(Wo, box[0]), _cdiv(Ho, box[1]), _cdiv(Do, box[2]), _cdiv(N, box[3]))
    n_tiles = grid_t[0] * grid_t[1] * grid_t[2] * grid_t[3]
    aw = min(cin, 64)
    per_slice, chunks = 128 // aw, cin // aw
    n_tile = min(cout, 128)
    n_blocks = cout // n_tile
    slices = _cdiv(taps * chunks, per_slice)
    splits = max(1, min(_cdiv(2 * sms, slices * n_blocks), n_tiles))
    tpc = _cdiv(n_tiles, splits)
    n_splits = _cdiv(n_tiles, tpc)
    return dict(n_tile=n_tile, box=box, tiles=grid_t, n_tiles=n_tiles, slices=slices, per_slice=per_slice,
                last_slice_atoms=taps * chunks - (slices - 1) * per_slice, n_splits=n_splits, tiles_per_cta=tpc,
                last_split=n_tiles - (n_splits - 1) * tpc)


def tile_index(N, Do, Ho, Wo, tile, device='cpu'):
    """(N, Do, Ho, Wo) int64: the linear index (w fastest, then h, d, image) of the output tile holding each pixel, the
    order both conv_tma kernels walk their tiles in."""
    tw, th, td, tn = tile
    i = [torch.arange(s, device=device) // t for s, t in zip((N, Do, Ho, Wo), (tn, td, th, tw))]
    nw, nh, nd = _cdiv(Wo, tw), _cdiv(Ho, th), _cdiv(Do, td)
    return ((i[0].view(-1, 1, 1, 1) * nd + i[1].view(1, -1, 1, 1)) * nh + i[2].view(1, 1, -1, 1)) * nw + i[3].view(1, 1, 1, -1)


# ------------------------------------------------------------------------------------------------ dense faults
def _one_tap(w, t):
    """w with every filter tap but the t-th (row-major over the kernel window) zeroed."""
    m = torch.zeros(w[0, 0].numel(), dtype=w.dtype, device=w.device)
    m[t] = 1
    return w * m.view(w.shape[2:])


def _px(t):
    """(N, C, *S) -> (N, D, H, W, C) so 2-D and 3-D outputs index alike."""
    return (t.unsqueeze(2) if t.dim() == 4 else t).movedim(1, -1)


def conv_fwd_faults(out, pre, x, w, stride, pad, relu, tile):
    """Copies of a correct forward output (N, Cout, *S) with one fault each: filter tap 0 (the corner tap, the one the
    zero padding clips most) dropped, output channels 0 and 1 swapped, and the last output tile (of the last N_TILE
    channel block) left at zero. `pre` is the float64 reference before the activation."""
    conv = _conv_ops(w.dim() - 2)[0]
    act = (lambda t: t.clamp(min=0)) if relu else (lambda t: t)
    drop = act(pre - conv(x.double(), _one_tap(w, 0).double(), None, stride, pad)).to(out.dtype)
    swapped = out.clone()
    swapped[:, [0, 1]] = out[:, [1, 0]]
    o = _px(out)
    idx = tile_index(*o.shape[:4], tile, out.device)
    tail = out.clone()
    _px(tail)[..., -min(out.shape[1], 128):][idx == idx.max()] = 0
    return [('filter tap 0 dropped', drop), ('output channels 0 and 1 swapped', swapped),
            ('last output tile left at zero', tail)]


def conv_dgrad_faults(out, ref, dy, w, x_shape, stride, pad, tile=None):
    """A correct dgrad with filter tap 0 dropped, input channels 0 and 1 swapped, and, at stride 2, one parity class left
    at zero: (1, 1), the smallest one for odd extents, or (0, 0) for a 1-wide filter (the only class any tap reaches); at
    stride 1 the last tile (`tile`, of the last channel block)."""
    dgrad = _conv_ops(w.dim() - 2)[1]
    drop = (ref - dgrad(x_shape, _one_tap(w, 0).double(), dy.double(), stride, pad)).to(out.dtype)
    swapped = out.clone()
    swapped[:, [0, 1]] = out[:, [1, 0]]
    faults = [('filter tap 0 dropped', drop), ('input channels 0 and 1 swapped', swapped)]
    hole = out.clone()
    if stride == 2:
        p = 0 if w.shape[-1] == 1 else 1
        hole[..., p::2, p::2] = 0
        faults.append((f'parity class ({p}, {p}) left at zero', hole))
    else:
        idx = tile_index(*_px(out).shape[:4], tile, out.device)
        _px(hole)[..., -min(out.shape[1], 128):][idx == idx.max()] = 0
        faults.append(('last output tile left at zero', hole))
    return faults


def wgrad_split_faults(out, x, dy, w_shape, stride, pad, geom):
    """A correct weight gradient without the pixel tiles of its last (shortest) split."""
    wgrad = _conv_ops(len(w_shape) - 2)[2]
    d = _px(dy)
    split = tile_index(*d.shape[:4], geom['box'], dy.device) // geom['tiles_per_cta']
    keep = (split == split.max()).to(dy.dtype)
    dym = dy * (keep if dy.dim() == 5 else keep[:, 0]).unsqueeze(1)
    part = wgrad(x.double(), w_shape, dym.double(), stride, pad)
    return [(f'pixel split {int(split.max())} ({geom["last_split"]} tiles) dropped', (out.double() - part).to(out.dtype))]


def direct_wgrad_slice_faults(out, x, dy, w_shape, stride, pad, slice_len):
    """A correct direct-kernel weight gradient without its last pixel slice (output pixels m >= (slices - 1) slice_len in
    the (image, row, column) order of conv2d_direct_wgrad_kernel; bf16_bounds.direct_wgrad_slices)."""
    wgrad = _conv_ops(2)[2]
    N, _, Ho, Wo = dy.shape
    m = torch.arange(N * Ho * Wo, device=dy.device).view(N, 1, Ho, Wo)
    first = (N * Ho * Wo - 1) // slice_len * slice_len
    part = wgrad(x.double(), w_shape, (dy.double() * (m >= first)), stride, pad)
    return [(f'pixel slice at {first} dropped', (out.double() - part).to(out.dtype))]


def attn_fwd_faults(o, q, k, v, key_pad, scale):
    """A correct attention output with one padded key treated as live (of the scans with live keys, the padded key with
    the largest values: the tests give padded keys large values so that a leak is visible), and with
    the keys of the last partial 128-key tile dropped."""
    Lk = k.shape[2]
    assert Lk % 128, 'the last key tile must be partial'
    faults = []
    some_live = ~key_pad.all(1, keepdim=True)
    size = v.double().abs().sum((1, 3)).masked_fill(~(key_pad & some_live), -1.0)
    if float(size.max()) >= 0:
        b, j = divmod(int(torch.argmax(size)), Lk)
        leak = key_pad.clone()
        leak[b, j] = False
        faults.append(('a padded key treated as live', attn_ref(q, k, v, leak, scale)['o'][0].to(o.dtype)))
    cut = key_pad.clone()
    cut[:, Lk // 128 * 128:] = True
    faults.append(('the last partial key tile dropped', attn_ref(q, k, v, cut, scale)['o'][0].to(o.dtype)))
    return faults


def attn_dq_faults(dq, k, dS):
    """A correct dQ without the partial of one 128-key tile (the one with the largest partial: where padding leaves a
    tile few live keys, its partial may be below the bound's resolution)."""
    parts = [dS[..., t0:t0 + 128] @ k[:, :, t0:t0 + 128].double() for t0 in range(0, k.shape[2], 128)]
    j = max(range(len(parts)), key=lambda i: float(parts[i].abs().sum()))
    return [(f'the dQ partial of key tile {j} dropped', (dq.double() - parts[j]).to(dq.dtype))]


# ------------------------------------------------------------------------------------------------ autograd references
def bilinear_ref(op, x, w, dy):
    """For an operation `op(x, w)` linear in each operand (a convolution, a transposed convolution): float64 y, dx, dw by
    autograd, each with its A (the same computation on |x|, |w|, |dy|). Returns {'y': (y, A), 'dx': ..., 'dw': ...}."""
    out = {}
    for tag, (xs, ws, ds) in (('v', (x.double(), w.double(), dy.double())),
                              ('a', (x.double().abs(), w.double().abs(), dy.double().abs()))):
        xs, ws = xs.requires_grad_(True), ws.requires_grad_(True)
        y = op(xs, ws)
        dx, dw = torch.autograd.grad(y, (xs, ws), ds)
        out[tag] = (y.detach(), dx, dw)
    return {k: (out['v'][i], out['a'][i]) for i, k in enumerate(('y', 'dx', 'dw'))}


# ------------------------------------------------------------------------------------------------ point painting
def paint_ref(feat, pts, batch, tx, ty, front, pad_hw, dout=None, dtype=torch.float64):
    """Point painting (csrc/paint.cu) on the geometry the tests build: every view v of scan b is a pure translation,
    u = x + tx[b, v], v = y + ty[b, v] at depth 1 (front[b, v]) or behind the camera (Z < 0: the point projects outside the
    map), and the feature map is sampled at the nearest pixel round(u), round(v) (the padded extent is (Hf - 1, Wf - 1), so
    grid_sample's align_corners scaling is the identity; the tests keep u, v an odd multiple of 1/8 from any pixel boundary,
    so the selection is exact in any arithmetic). As in the kernel, the sum runs over every view whose pixel is inside the
    map, the divisor counts the views with 0 < u < pad_w, 0 < v < pad_h in front of the camera.
    feat (B*V, Hf, Wf, C) channels-last; pts (N, 3); batch (N,) scan of each point. Returns (out (N, C), A, n_red) and,
    with `dout`, (dfeat (B*V*Hf*Wf, C), A, n_red): dfeat[pixel] = sum over (point, view) pairs at that pixel of
    dout[point] / count[point]. Also returns the (N, V) hit / valid masks and pixel rows for the fault builders."""
    BV, Hf, Wf, C = feat.shape
    V = tx.shape[1]
    u = pts[:, 0:1].double() + tx[batch.long()].double()
    v = pts[:, 1:2].double() + ty[batch.long()].double()
    fr = front[batch.long()]
    ix, iy = torch.floor(u + 0.5).long(), torch.floor(v + 0.5).long()
    hit = fr & (ix >= 0) & (ix < Wf) & (iy >= 0) & (iy < Hf)
    valid = fr & (u > 0) & (u < pad_hw[1]) & (v > 0) & (v < pad_hw[0])
    count = valid.sum(1, keepdim=True).to(dtype)
    inv = torch.where(count > 0, 1 / count, torch.zeros_like(count))
    img = batch.long()[:, None] * V + torch.arange(V, device=feat.device)[None]
    row = torch.where(hit, (img * Hf + iy.clamp(0, Hf - 1)) * Wf + ix.clamp(0, Wf - 1), 0)
    f = feat.reshape(BV * Hf * Wf, C).to(dtype)
    g = f[row] * hit[..., None]                                         # (N, V, C)
    res = dict(fwd=(g.sum(1) * inv, g.abs().sum(1) * inv, V + 2), hit=hit, valid=valid, row=row, inv=inv)
    if dout is not None:
        d = dout.to(dtype) * inv
        pr, pd = row[hit], d[:, None, :].expand(-1, V, -1)[hit]
        df = torch.zeros((BV * Hf * Wf, C), dtype=dtype, device=feat.device).index_add_(0, pr, pd)
        A = torch.zeros_like(df).index_add_(0, pr, pd.abs())
        n = torch.zeros((BV * Hf * Wf, 1), dtype=dtype, device=feat.device).index_add_(
            0, pr, torch.ones((pr.shape[0], 1), dtype=dtype, device=feat.device))
        res['bwd'] = (df, A, n + 1)
    return res


def paint_faults(out, dfeat, ref, feat, dout):
    """Painting outputs with one fault each. Forward: view j of every scan dropped (j the view that sees the most
    points); the divisor counting every view whose pixel is inside the map (not only the valid ones); channels 0 and 1
    swapped. Backward: the pairs of view j dropped; the same divisor fault."""
    hit, valid, row, inv = ref['hit'], ref['valid'], ref['row'], ref['inv']
    N, V = hit.shape
    C = feat.shape[-1]
    f = feat.reshape(-1, C).double()
    j = int(torch.argmax(hit.sum(0)))
    g0 = f[row[:, j]] * hit[:, j:j + 1] * inv
    cnt = hit.sum(1, keepdim=True).double()
    wrong = (f[row] * hit[..., None]).sum(1) / cnt.clamp(min=1)
    sw = out.clone()
    sw[:, [0, 1]] = out[:, [1, 0]]
    fwd = [(f'views {j} dropped', (out.double() - g0).to(out.dtype)),
           ('divisor counts every view inside the map', wrong.to(out.dtype)), ('channels 0 and 1 swapped', sw)]
    d = dout.double() * inv
    bad0 = dfeat.double().index_add(0, row[:, j][hit[:, j]], -d[hit[:, j]])
    d_wrong = dout.double() / cnt.clamp(min=1)
    pr = row[hit]
    bad1 = torch.zeros_like(dfeat, dtype=torch.float64).index_add_(0, pr, d_wrong[:, None, :].expand(-1, V, -1)[hit])
    bwd = [(f'pairs of views {j} dropped', bad0.to(dfeat.dtype)),
           ('divisor counts every view inside the map', bad1.to(dfeat.dtype))]
    return fwd, bwd


# ================================================================================================ head, loss, elementwise
# The remaining floating-point kernels of the bf16 steps (tests/test_head_elementwise_bf16_gpu.py): the sigmoid focal loss,
# the 2-D backbone's bias + residual + activation epilogue and its backward, and the interpolation of `_prune`. The others
# of that module (gather2_rows, img_normalize, cast) are held bit for bit.
FLT_MIN = 1.17549435e-38
LOG_FLT_MIN = math.log(FLT_MIN)
FOCAL_ELEM = 64


def focal_ref(x, target, row_w, gamma, alpha, scale=1.0):
    """mmcv's sigmoid focal loss (csrc/head.cu) in float64 on the same logits x (n, C): per element
      positive (target[r] == c): l = -alpha (1-p)^gamma log(max(p, FLT_MIN)),
                                 g = -alpha (1-p)^gamma (1 - p - gamma p log(max(p, FLT_MIN)))
      negative:                  l = -(1-alpha) p^gamma log(max(1-p, FLT_MIN)),
                                 g = -(1-alpha) p^gamma (gamma (1-p) log(max(1-p, FLT_MIN)) - p)
    each times row_w[r] (and g times `scale`). A target outside [0, C) (-1 or >= C) has no positive column.

    Conditioning: the kernel evaluates p = 1 / (1 + expf(-x)) to a few fp32 roundings of p, and 1 - p in fp32 inherits that
    absolute error, i.e. a relative error of (p / (1 - p)) 2^-24 = e^x 2^-24 per rounding; (1-p)^gamma, and log p near
    p = 1 (magnitude ~ e^-x), carry it into the element. At the other end, x << 0, 1 - p is accurate but near 1, and
    logf(1 - p) (magnitude ~ p ~ e^x) is off by the absolute rounding of 1 - p, a relative 2^-24 e^-x. So an element is off
    by a relative 2^-24 FOCAL_ELEM K(x) with K(x) = 1 + e^|x|; FOCAL_ELEM = 64 covers the ~10 roundings of an element
    (expf's 2 ulp included) with each term's conditioning. Returns dict(l, g, K) in float64."""
    xd = x.double()
    p, q = torch.sigmoid(xd), torch.sigmoid(-xd)             # q = 1 - p without cancellation
    C = x.shape[1]
    pos = target.view(-1, 1).to(x.device) == torch.arange(C, device=x.device).view(1, -1)
    lp, lq = torch.log(p.clamp(min=FLT_MIN)), torch.log(q.clamp(min=FLT_MIN))
    l = torch.where(pos, -alpha * q ** gamma * lp, -(1 - alpha) * p ** gamma * lq)
    g = torch.where(pos, -alpha * q ** gamma * (q - gamma * p * lp), -(1 - alpha) * p ** gamma * (gamma * q * lq - p))
    w = row_w.double().view(-1, 1)
    return dict(l=l * w, g=g * w * scale, K=1 + torch.exp(xd.abs()))


def focal_operands(n, C, gen, wide=False):
    """Logits (n, C) fp32, targets (n,) int64 and row weights (n,) fp32 for the focal cases. Targets: a third -1, a third
    >= C (no positive either way), a third in range. Row weights of unequal size from 0.05 to 1, the last row 40 (so the
    last, partial, block of the sum carries weight). 'typical' logits are those of a training head: negatives N(-2, 2)
    within [-12, 6], positives N(3, 2) within [-4, 12]; wide=True draws every logit uniformly from [-12, 12], which puts
    negatives where the fp32 1 - p is worst conditioned (K up to e^12)."""
    kind = torch.randint(0, 3, (n, ), generator=gen)
    target = torch.where(kind == 0, -1, torch.where(kind == 1, C + torch.randint(0, 5, (n, ), generator=gen),
                                                    torch.randint(0, C, (n, ), generator=gen)))
    if wide:
        x = torch.rand(n, C, generator=gen) * 24 - 12
    else:
        x = (torch.randn(n, C, generator=gen) * 2 - 2).clamp(-12, 6)
        pos = torch.nonzero(kind == 2).squeeze(1)
        x[pos, target[pos]] = (torch.randn(pos.numel(), generator=gen) * 2 + 3).clamp(-4, 12)
    w = torch.rand(n, generator=gen) * 0.95 + 0.05
    w[-1] = 40.0
    return x, target.long(), w


def focal_sum_bound(ref, n_blocks):
    """(sum, A) of the focal loss sum for the bound with n_red = 1: each element rounded as focal_ref says, then added
    through the 256-wide block (5 shuffle levels, 8 warp partials) and the ordered sum of the n_blocks partials."""
    la = ref['l'].abs()
    return ref['l'].sum(), (5 + 8 + n_blocks) * la.sum() + FOCAL_ELEM * (ref['K'] * la).sum()


def focal_faults_fwd(x, target, row_w, gamma, alpha, total):
    """Copies of a correct loss sum `total` with one fault each: alpha swapped between the classes, the row with the
    largest contribution dropped, the last partial 256-element block dropped, gamma taken as 1, and (C > 1) the positive
    column off by one."""
    n, C = x.shape
    ref = focal_ref(x, target, row_w, gamma, alpha)['l']
    t1 = torch.where((target >= 0) & (target < C - 1), target + 1, target)
    row = ref.sum(1)
    last = n * C // 256 * 256
    assert last < n * C, 'the last block must be partial'
    d = total.double()
    faults = [('alpha swapped', d - ref.sum() + focal_ref(x, target, row_w, gamma, 1 - alpha)['l'].sum()),
              ('largest row dropped', d - row[row.abs().argmax()]),
              ('last partial block dropped', d - ref.reshape(-1)[last:].sum()),
              ('gamma taken as 1', d - ref.sum() + focal_ref(x, target, row_w, 1.0, alpha)['l'].sum())]
    if C > 1:
        faults.append(('positive column off by one', d - ref.sum() + focal_ref(x, t1, row_w, gamma, alpha)['l'].sum()))
    return faults


def focal_faults_bwd(x, target, row_w, gamma, alpha, scale, grad):
    """A correct focal gradient with: alpha swapped, the row weights dropped, gamma taken as 1, the sign flipped, `scale`
    ignored and (C > 1) the positive column off by one."""
    C = x.shape[1]
    t1 = torch.where((target >= 0) & (target < C - 1), target + 1, target)
    f = lambda **kw: focal_ref(x, kw.get('t', target), kw.get('w', row_w), kw.get('gm', gamma), kw.get('a', alpha),  # noqa: E731
                               kw.get('s', scale))['g'].to(grad.dtype)
    faults = [('alpha swapped', f(a=1 - alpha)), ('row weights dropped', f(w=torch.ones_like(row_w))),
              ('gamma taken as 1', f(gm=1.0)), ('sign flipped', -grad), ('scale ignored', f(s=1.0))]
    return faults + ([('positive column off by one', f(t=t1))] if C > 1 else [])


def _act(z, act):
    return z if act == 0 else (z.clamp(min=0) if act == 1 else torch.where(z > 0, z, torch.expm1(z)))


def bias_act_ref(x, bias, res, act):
    """y = act(x + bias[c] (+ res)) in float64 on (rows, C): (y, A, n_red). The kernel rounds the two additions (and
    expm1f for ELU), and the output rounding applies to a value already off by those: n_red = 3 (ELU 4). Every activation
    is 1-Lipschitz, so the error of z carries over to y. (One fp32 rounding of x + b alone needs c n_red <= 1: the fp32
    cases measured 0.42 at n_red = 2.)"""
    z = x.double() + bias.double().view(1, -1)
    A = x.double().abs() + bias.double().abs().view(1, -1)
    if res is not None:
        z, A = z + res.double(), A + res.double().abs()
    return _act(z, act), A, 4 if act == 2 else 3


def bias_act_faults(y, x, bias, res, act, rows_per_block):
    """The epilogue with the bias read one channel off, the residual dropped (when there is one), ELU / ReLU left out, and
    the last partial block of rows not written (in place: still holding x)."""
    dt = y.dtype
    faults = [('bias one channel off', bias_act_ref(x, bias.roll(1), res, act)[0].to(dt))]
    if res is not None:
        faults.append(('residual dropped', bias_act_ref(x, bias, None, act)[0].to(dt)))
    if act:
        faults.append(('activation left out', bias_act_ref(x, bias, res, 0)[0].to(dt)))
    tail = y.clone()
    r0 = x.shape[0] // rows_per_block * rows_per_block
    if r0 == x.shape[0]:
        r0 -= rows_per_block
    tail[r0:] = x[r0:]
    faults.append(('last block of rows not written', tail))
    return faults


def act_bwd_ref(dy, z, y, act):
    """dx = dy act'(z) in float64, the derivative from the float64 pre-activation z, for the kernel that reads it from the
    stored output y (ReLU: y > 0; ELU: y > 0 ? 1 : y + 1). Returns (dx, A, n_red, fixed): the product rounds once (ELU: y + 1
    too); `fixed` = |dy| |y - act(z)| (1 + 2^-7) is what reading the derivative from the rounded output y costs (ELU's
    derivative is y + 1 on the negative side, so it is off by exactly the error of y; on the positive side it is 1 either
    way; ReLU's is exact while y and z have the same sign), the factor keeping the output rounding of a value already off by
    that much covered."""
    zd, dyd = z.double(), dy.double()
    d = torch.ones_like(zd) if act == 0 else ((zd > 0).double() if act == 1 else torch.where(zd > 0, 1.0, torch.exp(zd)))
    dx = dyd * d
    fixed = dyd.abs() * (y.double() - _act(zd, act)).abs() * (zd <= 0) * (1 + 2.0 ** -7) if act == 2 else \
        torch.zeros_like(dx)
    return dx, dx.abs() + fixed, 2 if act == 2 else 1, fixed


def act_bwd_faults(dx, dy, z, act):
    """The activation gradient with the tail (the last n % 8 elements, or the last 8) not written, ELU's derivative taken
    as ReLU's, and the sign flipped."""
    n = dx.numel()
    tail = dx.clone()
    tail[n - (n % 8 or 8):] = 0
    faults = [('tail not written', tail), ('sign flipped', -dx)]
    if act == 2:
        faults.append(('ReLU derivative for ELU', (dy.double() * (z.double() > 0)).to(dx.dtype)))
    return faults


def seg_norm_bwd_fixed(x, F, st):
    """How far seg_norm_bwd_ref's dx, dgamma and dbeta move when gy moves by at most F per element (gamma excluded from
    dx: multiply by |gamma|): rstd (F + mean_s F + |xhat| mean_s(F |xhat|)), sum F |xhat|, sum F."""
    seg, n, rs = st['seg'], st['n'], st['rs']
    S, C = n.shape[0], x.shape[1]
    xh = ((x.double() - st['mean'][seg]) * rs[seg]).abs()
    P = torch.zeros((S, C), dtype=torch.float64, device=x.device)
    mf, mfx = P.clone().index_add_(0, seg, F) / n, P.clone().index_add_(0, seg, F * xh) / n
    return rs[seg] * (F + mf[seg] + xh * mfx[seg]), (F * xh).sum(0), F.sum(0)


def interp_ref(coords, feats, ts, query, trunc=False):
    """Multilinear interpolation (csrc/hash.cu::interp_features_kernel) in float64 on the same features: coords (n, 4)
    int64 [b, x, y, z] (multiples of ts), feats (n, C), query (m, 4) int64. base = floor(q / ts) ts, frac = q / ts - floor,
    out = sum over the 8 corners present of F[corner] w_k, w_k = product of frac or 1 - frac. Returns (out, A, n_red = 11:
    eight products and additions plus the three roundings of a weight, the (m, 8) corner rows (-1 when absent), the (m, 8)
    weights). trunc=True rounds q / ts towards zero instead (a fault)."""
    import numpy as np
    q = np.asarray(query, dtype=np.int64)
    c = np.asarray(coords, dtype=np.int64)
    v = q[:, 1:] / float(ts)
    fl = np.trunc(v) if trunc else np.floor(v)
    base = fl.astype(np.int64) * ts
    frac = v - fl
    off = 1 << 20

    def key(a):
        return ((a[:, 0] * (1 << 21) + a[:, 1] + off) * (1 << 21) + a[:, 2] + off) * (1 << 21) + a[:, 3] + off
    order = np.argsort(key(c))
    ks = key(c)[order]
    rows = np.full((q.shape[0], 8), -1, dtype=np.int64)
    w = np.zeros((q.shape[0], 8))
    for k in range(8):
        d = np.array([k & 1, (k >> 1) & 1, (k >> 2) & 1])
        kk = key(np.concatenate([q[:, :1], base + d * ts], 1))
        pos = np.clip(np.searchsorted(ks, kk), 0, len(ks) - 1)
        rows[:, k] = np.where(ks[pos] == kk, order[pos], -1)
        w[:, k] = np.prod(np.where(d.astype(bool), frac, 1 - frac), 1)
    f = feats.double()
    r = torch.from_numpy(rows).to(f.device)
    wt = torch.from_numpy(w).to(f.device)
    g = f[r.clamp(min=0)] * (r >= 0)[..., None] * wt[..., None]
    return g.sum(1), g.abs().sum(1), 11, r, wt


def interp_faults(out, coords, feats, ts, query):
    """The interpolation with the last corner (k = 7) dropped, q / ts truncated towards zero instead of floored, and absent
    corners read as row 0."""
    ref, _, _, rows, wt = interp_ref(coords, feats, ts, query)
    f = feats.double()
    k7 = ref - f[rows[:, 7].clamp(min=0)] * ((rows[:, 7] >= 0) * wt[:, 7])[:, None]
    absent = ref + ((rows < 0) * wt).sum(1, keepdim=True) * f[0][None]
    return [('corner 7 dropped', k7.to(out.dtype)),
            ('truncation instead of floor', interp_ref(coords, feats, ts, query, trunc=True)[0].to(out.dtype)),
            ('absent corners read as row 0', absent.to(out.dtype))]
