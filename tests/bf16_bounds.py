"""Per-element error bounds for the bf16 kernels of the sparse branch, their float64 references, and the faults the bounds
must catch.

A kernel output `out` (bf16 operands, fp32 accumulation) is checked element by element against a float64 reference `ref`
computed from the same bf16-rounded operands:

    |out - ref| <= out_rel * |ref| + c * 2^-24 * n_red * A

`out_rel` is one rounding of the output type (2^-8 for bf16 outputs: twice round-to-nearest's 2^-9; 2^-24 for fp32 outputs)
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

Nothing here imports the library: it runs on CPU tensors as well as CUDA tensors.
"""
import math

import torch

U32 = 2.0 ** -24
OUT_REL_BF16 = 2.0 ** -8
OUT_REL_F32 = 2.0 ** -24
C_ACC = 0.5


# ------------------------------------------------------------------------------------------------ the bound
def excess_ratio(out, ref, A, n_red, out_rel):
    """The smallest c for which `out` passes: max over elements of (|out - ref| - out_rel |ref|)+ / (2^-24 n_red A).
    inf when an element whose bound is exactly zero (ref = A = 0) is not exactly zero, or when `out` holds a NaN."""
    err = (out.double() - ref).abs()
    excess = (err - out_rel * ref.abs()).clamp(min=0)
    if torch.isnan(err).any():
        return math.inf
    scale = U32 * n_red * A
    scale = torch.broadcast_to(torch.as_tensor(scale, dtype=torch.float64, device=ref.device), excess.shape)
    if bool(((excess > 0) & (scale == 0)).any()):
        return math.inf
    r = torch.where(excess > 0, excess / torch.where(scale > 0, scale, 1.0), torch.zeros_like(excess))
    return float(r.max()) if r.numel() else 0.0


def within(out, ref, A, n_red, out_rel, c=C_ACC):
    err = (out.double() - ref).abs()
    return bool((err <= out_rel * ref.abs() + c * U32 * n_red * A).all())


def assert_within(out, ref, A, n_red, out_rel, what):
    """Assert the bound at C_ACC; returns the ratio the output needed (reported by the tests)."""
    r = excess_ratio(out, ref, A, n_red, out_rel)
    assert within(out, ref, A, n_red, out_rel), f'{what}: needs c = {r:.3g} > C_ACC = {C_ACC}'
    return r


def assert_rejects(faults, ref, A, n_red, out_rel):
    """Every faulty copy of a correct output must fail the bound, else the bound is too loose to see that fault."""
    passed = [name for name, bad in faults if within(bad, ref, A, n_red, out_rel)]
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


# ------------------------------------------------------------------------------------------------ faults
def conv_faults(out, x, w, nbr, w_layout=1, tile_rows=128):
    """Copies of a correct gather-GEMM output with one fault each, as a tile kernel could make them:
    the contribution of the sparsest used kernel offset missing, output channels 0 and 1 swapped, the last 64-channel
    slice of the reduction missing, and the last (partial) 128-row tile left at zero."""
    K, n_out = nbr.shape
    assert n_out % tile_rows, 'the last row tile must be partial'
    cin = x.shape[1]
    used = [(int((nbr[k] >= 0).sum()), k) for k in range(K) if bool((nbr[k] >= 0).any())]
    k_min = min(used)[1]
    one = torch.full_like(nbr, -1)
    one[k_min] = nbr[k_min]
    drop_k = gather_gemm(x, w, one, w_layout)[0]
    xs = x.clone()
    xs[:, :cin - 64] = 0
    drop_slice = gather_gemm(xs, w, nbr, w_layout)[0]
    swapped = out.clone()
    swapped[:, [0, 1]] = out[:, [1, 0]]
    tail = out.clone()
    tail[n_out // tile_rows * tile_rows:] = 0
    return [(f'kernel offset {k_min} dropped', (out.double() - drop_k).to(out.dtype)),
            ('output channels 0 and 1 swapped', swapped),
            (f'reduction channels {cin - 64}..{cin - 1} zeroed', (out.double() - drop_slice).to(out.dtype)),
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


def random_kernel_map(n_in, n_out, K, gen, device='cpu', empty_offset=None, single_offset=None, empty_tile=None):
    """nbr (K, n_out) int32: through each offset an injective map into [0, n_in) of random density (as a real kernel map
    is); `empty_offset` gets no neighbour at all, `single_offset` exactly one, and the 128 rows of `empty_tile` none."""
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
        nbr[:, empty_tile * 128:(empty_tile + 1) * 128] = -1
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
