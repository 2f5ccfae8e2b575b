"""The per-element bf16 bound of tests/bf16_bounds.py (used by test_sparse_bf16_gpu.py) on CPU: a bf16-emulated correct
output (fp32 accumulation, one bf16 rounding) passes it, and every fault it is meant to see is rejected at C_ACC."""
import torch

import bf16_bounds as B


def test_bound_accepts_emulated_conv_and_rejects_its_faults():
    gen = torch.Generator().manual_seed(0)
    n_in, n_out, K, cin, cout = 400, 300, 27, 128, 64
    nbr = B.random_kernel_map(n_in, n_out, K, gen, empty_offset=5, single_offset=7, empty_tile=1)
    for w_layout in (1, 0):
        x = torch.randn(n_in, cin, generator=gen).bfloat16()
        w = (torch.randn((K, cin, cout) if w_layout else (K, cout, cin), generator=gen) / (K * cin) ** 0.5).bfloat16()
        ref, A, n_red = B.gather_gemm(x, w, nbr, w_layout)
        out = B.gather_gemm(x, w, nbr, w_layout, dtype=torch.float32)[0].bfloat16()
        B.assert_within(out, ref, A, n_red, B.OUT_REL_BF16, f'emulated conv, layout {w_layout}')
        assert bool((out[128:256] == 0).all())
        faults = B.conv_faults(out, x, w, nbr, w_layout)
        assert len(faults) == 4
        B.assert_rejects(faults, ref, A, n_red, B.OUT_REL_BF16)


def test_bound_accepts_emulated_wgrad_and_rejects_a_dropped_chunk():
    gen = torch.Generator().manual_seed(1)
    cp, n_rows, cin, cout = 512, 1300, 64, 64
    pin, pout, koff = B.random_pairs([0, cp - 1, cp, cp + 1, 40, 1200], n_rows, n_rows, gen)
    x = torch.randn(n_rows, cin, generator=gen).bfloat16()
    dy = torch.randn(n_rows, cout, generator=gen).bfloat16()
    ref, A, n_red = B.pair_wgrad(x, dy, pin, pout, koff)
    out = B.pair_wgrad(x, dy, pin, pout, koff, dtype=torch.float32)[0]
    B.assert_within(out, ref, A, n_red, B.OUT_REL_F32, 'emulated wgrad')
    faults = B.wgrad_faults(out, x, dy, pin, pout, koff, cp)
    assert '(1 pairs)' in faults[0][0]          # the tail chunk of the offset with chunk_pairs + 1 pairs: the smallest
    B.assert_rejects(faults, ref, A, n_red, B.OUT_REL_F32)


def test_bound_is_exact_where_every_term_is_zero():
    ref = torch.zeros(4, 3, dtype=torch.float64)
    A = torch.zeros_like(ref)
    out = torch.zeros(4, 3)
    assert B.excess_ratio(out, ref, A, 10, B.OUT_REL_BF16) == 0.0 and B.within(out, ref, A, 10, B.OUT_REL_BF16)
    out[2, 1] = 1e-30
    assert B.excess_ratio(out, ref, A, 10, B.OUT_REL_BF16) == float('inf')
    assert not B.within(out, ref, A, 10, B.OUT_REL_BF16)
    out[2, 1] = float('nan')
    assert not B.within(out, ref + 1, A + 1, 10, B.OUT_REL_BF16)


def test_selection_rules_follow_the_sm_count():
    assert B.tc_fwd_n_tile(128 * 132, 256, 132) == 256 and B.tc_fwd_n_tile(128 * 131, 256, 132) == 128
    assert B.tc_fwd_n_tile(128 * 66, 128, 132) == 64 and B.tc_fwd_n_tile(128 * 114, 256, 114) == 256
    assert B.tc_wgrad_chunk_pairs(27 * 3000, 192, 64, 132) == 512
    assert B.tc_wgrad_chunk_pairs(27 * 200000, 256, 128, 132) == 5120


def test_dense_selection_rules():
    assert B.conv_choose_tile(160, 120, 1, 2) == (32, 4, 1, 1)           # 128-pixel tiles that divide the output exactly
    assert B.conv_choose_tile(3, 3, 1, 100) == (3, 3, 1, 14)             # whole 3x3 images, 14 per tile
    assert B.conv_choose_tile(4, 4, 16, 1) == (4, 2, 16, 1)              # 3-D: TD > 1 (equal waste: the first found)
    g = B.conv_tma_geometry(2, 1, 120, 160, 2048, 132)
    assert g['n_tile'] == 128 and g['n_work'] == 300 * 16 and g['grid'] == 132 and not g['partial']
    w = B.wgrad_tma_geometry(64, 1, 3, 3, 64, 64, 9, 132)
    assert w['box'] == (4, 4, 1, 4) and w['slices'] == 5 and w['n_tiles'] == 16
    w = B.wgrad_tma_geometry(2, 1, 60, 80, 16, 16, 9, 132)
    assert w['per_slice'] == 8 and w['slices'] == 2 and w['last_slice_atoms'] == 1
    assert w['n_splits'] == _cdiv(w['n_tiles'], w['tiles_per_cta']) and 0 < w['last_split'] <= w['tiles_per_cta']
    idx = B.tile_index(2, 1, 5, 7, (4, 2, 1, 1))
    assert idx.shape == (2, 1, 5, 7) and int(idx.max()) == 2 * 3 * 2 - 1 and int(idx[0, 0, 4, 6]) == 5


def _cdiv(a, b):
    return -(-a // b)


def _emulated_conv(x, w, stride, pad, bias=None, res=None):
    """The convolution as a bf16 kernel computes it: fp32 accumulation on the bf16 operands, one bf16 rounding."""
    conv = torch.nn.functional.conv2d if w.dim() == 4 else torch.nn.functional.conv3d
    y = conv(x.float(), w.float(), bias, stride, pad)
    return (y + res.float() if res is not None else y).clamp(min=0).bfloat16()


def test_bound_accepts_emulated_dense_conv_and_rejects_its_faults():
    gen = torch.Generator().manual_seed(2)
    for dims, cin, cout, k, stride, pad, S in ((2, 32, 16, 3, 1, 1, (13, 21)), (2, 16, 32, 3, 2, 1, (15, 19)),
                                               (3, 16, 16, 3, 2, 1, (5, 7, 9))):
        n = 3
        x = torch.randn((n, cin) + S, generator=gen).bfloat16()
        w = (torch.randn((cout, cin) + (k, ) * dims, generator=gen) / (cin * k ** dims) ** 0.5).bfloat16()
        b = torch.randn(cout, generator=gen)
        y = _emulated_conv(x, w, stride, pad, b)
        pre, A, n_red = B.dense_conv_ref(x, w, stride, pad, b)
        B.assert_within(y, pre.clamp(min=0), A, n_red, B.OUT_REL_BF16, 'emulated conv')
        So = y.shape[2:]
        tile = B.conv_choose_tile(So[-1], So[-2], So[0] if dims == 3 else 1, n)
        faults = B.conv_fwd_faults(y, pre, x, w, stride, pad, True, tile)
        assert len(faults) == 3
        B.assert_rejects(faults, pre.clamp(min=0), A, n_red, B.OUT_REL_BF16)
        # dgrad: fp32 transposed convolution of the bf16 dy, one rounding
        dy = torch.randn(y.shape, generator=gen).bfloat16()
        ref, A, n_red = B.dense_dgrad_ref(dy, w, x.shape, stride, pad)
        dgrad = torch.nn.grad.conv2d_input if dims == 2 else torch.nn.grad.conv3d_input
        dx = dgrad(x.shape, w.float(), dy.float(), stride, pad).bfloat16()
        B.assert_within(dx, ref, A, n_red, B.OUT_REL_BF16, 'emulated dgrad')
        tile = B.conv_choose_tile(S[-1], S[-2], S[0] if dims == 3 else 1, n)
        B.assert_rejects(B.conv_dgrad_faults(dx, ref, dy, w, x.shape, stride, pad, tile), ref, A, n_red, B.OUT_REL_BF16)


def test_bound_rejects_a_dropped_wgrad_split_on_integer_operands():
    """On operands in {-1, 0, 1} the weight gradient is exact (assert_exact) and a dropped pixel split is a non-zero
    integer in some element: the bound rejects it, although at this reduction length it could not on random operands."""
    gen = torch.Generator().manual_seed(3)
    n, cin, cout, S = 8, 16, 32, (30, 40)
    geom = B.wgrad_tma_geometry(n, 1, *S, cin, cout, 9, 132)
    assert geom['n_splits'] >= 2
    x = B.ternary((n, cin) + S, 0.15, gen).bfloat16()
    dy = B.ternary((n, cout) + S, 0.15, gen).bfloat16()
    ref, A, n_red = B.dense_wgrad_ref(x, dy, (cout, cin, 3, 3), 1, 1)
    out = torch.nn.grad.conv2d_weight(x.float(), (cout, cin, 3, 3), dy.float(), 1, 1)
    B.assert_exact(out, ref, A, 'emulated wgrad', out_bf16=False)
    faults = B.wgrad_split_faults(out, x, dy, (cout, cin, 3, 3), 1, 1, geom)
    B.assert_rejects(faults, ref, A, n_red, B.OUT_REL_F32)


def _emulated_attention(q, k, v, pad, scale, do):
    """Attention as csrc/attn_tc.cu computes it, in fp32: P rounded to bf16 before P V and P^T dO (l from the unrounded
    p), O stored bf16 and read back for delta, dS^T rounded to bf16 for dK and dQ."""
    qf, kf, vf, dof = q.float(), k.float(), v.float(), do.float()
    s = scale * qf @ kf.transpose(-1, -2)
    s = s.masked_fill(pad[:, None, None, :], -float('inf'))
    m = s.amax(-1, keepdim=True)
    m = torch.where(torch.isfinite(m), m, torch.zeros_like(m))
    p = torch.exp(s - m)
    l = p.sum(-1, keepdim=True)
    inv = torch.where(l > 0, 1 / l, torch.zeros_like(l))
    o = ((p.bfloat16().float() @ vf) * inv).bfloat16()
    P = p * inv
    delta = (o.float() * dof).sum(-1, keepdim=True)
    dS = (P * (dof @ vf.transpose(-1, -2) - delta) * scale).bfloat16().float()
    dv = (P.bfloat16().float().transpose(-1, -2) @ dof).bfloat16()
    dk = (dS.transpose(-1, -2) @ qf).bfloat16()
    dq = dS @ kf
    return o, dq, dk, dv


def test_bound_accepts_emulated_attention_and_rejects_its_faults():
    gen = torch.Generator().manual_seed(4)
    Bn, H, Lq, Lk = 3, 2, 70, 300
    q, k, v, do = (torch.randn(Bn, H, L, 32, generator=gen).bfloat16() for L in (Lq, Lk, Lk, Lq))
    pad = torch.zeros(Bn, Lk, dtype=torch.bool)
    pad[0, 250:] = True
    pad[1, :40] = True
    pad[2] = True
    k[:, :, :40] *= 16                                  # padded keys with large values: a leak must be visible
    v[:, :, :40] = 1000.0
    scale = 32 ** -0.5
    ref = B.attn_ref(q, k, v, pad, scale, do)
    outs = dict(zip(('o', 'dq', 'dk', 'dv'), _emulated_attention(q, k, v, pad, scale, do)))
    for nm, out in outs.items():
        val, A, fixed = ref[nm]
        B.assert_within(out, val, A, 1, B.OUT_REL_F32 if nm == 'dq' else B.OUT_REL_BF16, f'emulated attention {nm}',
                        fixed=fixed)
        assert bool((out[2] == 0).all()), 'a scan without live keys must give exact zeros'
    assert bool((ref['lse'][2] == -float('inf')).all())
    val, A, fixed = ref['o']
    faults = B.attn_fwd_faults(outs['o'], q, k, v, pad, scale)
    assert len(faults) == 2
    B.assert_rejects(faults, val, A, 1, B.OUT_REL_BF16, fixed)
    val, A, fixed = ref['dq']
    B.assert_rejects(B.attn_dq_faults(outs['dq'], k, ref['dS']), val, A, 1, B.OUT_REL_F32, fixed)


def test_bound_accepts_emulated_painting_and_rejects_its_faults():
    """Painting as csrc/paint.cu computes it (fp32 sums of bf16 features, one bf16 rounding forward; fp32 backward) passes
    the bound of bf16_bounds.paint_ref, and each fault of paint_faults is rejected."""
    gen = torch.Generator().manual_seed(5)
    Bn, V, Hf, Wf, N, C = 2, 9, 12, 16, 400, 40
    tx = torch.randint(-3, 4, (Bn, V), generator=gen).double() + 0.125
    ty = torch.randint(-3, 4, (Bn, V), generator=gen).double() - 0.375
    front = torch.rand(Bn, V, generator=gen) > 0.2
    batch = torch.randint(0, Bn, (N, ), generator=gen)
    pts = torch.stack([torch.randint(-20, 4 * (Wf + 5), (N, ), generator=gen), torch.randint(-20, 4 * (Hf + 5), (N, ),
                      generator=gen), torch.zeros(N, dtype=torch.long)], 1).double() * 0.25
    feat = torch.randn(Bn * V, Hf, Wf, C, generator=gen).bfloat16()
    dout = torch.randn(N, C, generator=gen).bfloat16()
    pad = (Hf - 1.0, Wf - 1.0)
    ref = B.paint_ref(feat, pts, batch, tx, ty, front, pad, dout)
    emu = B.paint_ref(feat, pts, batch, tx, ty, front, pad, dout, dtype=torch.float32)
    assert bool((ref['hit'] & ~ref['valid']).any())
    out, dfeat = emu['fwd'][0].bfloat16(), emu['bwd'][0]
    B.assert_within(out, *ref['fwd'], B.OUT_REL_BF16, 'emulated paint fwd', c=B.C_PAINT)
    B.assert_within(dfeat, *ref['bwd'], B.OUT_REL_F32, 'emulated paint bwd', c=B.C_PAINT)
    fwd_f, bwd_f = B.paint_faults(out, dfeat, ref, feat, dout)
    assert len(fwd_f) == 3 and len(bwd_f) == 2
    B.assert_rejects(fwd_f, *ref['fwd'], B.OUT_REL_BF16, c=B.C_PAINT)
    B.assert_rejects(bwd_f, *ref['bwd'], B.OUT_REL_F32, c=B.C_PAINT)


# ------------------------------------------------------------------------------------------------ head and elementwise
def _emulated_focal(x, t, w, gamma, alpha, scale):
    """csrc/head.cu's focal element in fp32: p = 1 / (1 + exp(-x)), 1 - p in fp32, the clamp to FLT_MIN."""
    xf = x.float()
    p = 1 / (1 + torch.exp(-xf))
    q = 1 - p
    pos = t.view(-1, 1) == torch.arange(x.shape[1]).view(1, -1)
    lp, lq = torch.log(p.clamp(min=B.FLT_MIN)), torch.log(q.clamp(min=B.FLT_MIN))
    pg, qg = p ** gamma, q ** gamma
    l = torch.where(pos, -alpha * qg * lp, -(1 - alpha) * pg * lq) * w.view(-1, 1)
    g = torch.where(pos, -alpha * qg * (q - gamma * p * lp), -(1 - alpha) * pg * (gamma * q * lq - p))
    return l, g * scale * w.view(-1, 1)


def test_bound_accepts_emulated_focal_and_rejects_its_faults():
    gen = torch.Generator().manual_seed(6)
    n, C = 300, 284
    x, t, w = B.focal_operands(n, C, gen)
    x = x.bfloat16()
    l, g = _emulated_focal(x, t, w, 2.0, 0.25, 0.37)
    ref = B.focal_ref(x, t, w, 2.0, 0.25, 0.37)
    n_blocks = (n * C + 255) // 256
    total, A = B.focal_sum_bound(ref, n_blocks)
    out = l.sum()
    B.assert_within(out, total, A, 1, B.OUT_REL_F32, 'emulated focal sum')
    B.assert_rejects(B.focal_faults_fwd(x, t, w, 2.0, 0.25, out), total, A, 1, B.OUT_REL_F32)
    gb = g.bfloat16()
    Ag = ref['K'] * ref['g'].abs()
    B.assert_within(gb, ref['g'], Ag, B.FOCAL_ELEM, B.OUT_REL_BF16, 'emulated focal grad')
    B.assert_rejects(B.focal_faults_bwd(x, t, w, 2.0, 0.25, 0.37, gb), ref['g'], Ag, B.FOCAL_ELEM, B.OUT_REL_BF16)
    xw = B.focal_operands(n, C, gen, wide=True)[0].bfloat16()      # the wide range: elementwise bound and faults
    gw = _emulated_focal(xw, t, w, 2.0, 0.25, 0.37)[1].bfloat16()
    ref = B.focal_ref(xw, t, w, 2.0, 0.25, 0.37)
    Ag = ref['K'] * ref['g'].abs()
    B.assert_within(gw, ref['g'], Ag, B.FOCAL_ELEM, B.OUT_REL_BF16, 'emulated focal grad, wide logits')
    B.assert_rejects(B.focal_faults_bwd(xw, t, w, 2.0, 0.25, 0.37, gw), ref['g'], Ag, B.FOCAL_ELEM, B.OUT_REL_BF16)


def test_bound_accepts_emulated_bias_act_and_act_bwd():
    gen = torch.Generator().manual_seed(7)
    rows, C = 301, 16
    for act in (0, 1, 2):
        x = torch.randn(rows, C, generator=gen).bfloat16()
        b = torch.randn(C, generator=gen)
        r = torch.randn(rows, C, generator=gen).bfloat16()
        z = x.float() + b + r.float()
        y = B._act(z, act).bfloat16()
        ref, A, n_red = B.bias_act_ref(x, b, r, act)
        B.assert_within(y, ref, A, n_red, B.OUT_REL_BF16, f'emulated bias act {act}')
        B.assert_rejects(B.bias_act_faults(y, x, b, r, act, 256 * 8 // C), ref, A, n_red, B.OUT_REL_BF16)
        dy = torch.randn(rows * C, generator=gen).bfloat16()
        zf = z.reshape(-1)
        yf = y.reshape(-1)
        d = torch.ones_like(zf) if act == 0 else ((yf > 0).float() if act == 1 else torch.where(yf > 0, 1.0, yf.float() + 1))
        dx = (dy.float() * d).bfloat16()
        ref, A, n_red, fixed = B.act_bwd_ref(dy, zf, yf, act)
        B.assert_within(dx[:-3], ref[:-3], A[:-3], n_red, B.OUT_REL_BF16, f'emulated act bwd {act}', fixed=fixed[:-3])
        B.assert_rejects(B.act_bwd_faults(dx[:-3], dy[:-3], zf[:-3], act), ref[:-3], A[:-3], n_red, B.OUT_REL_BF16,
                         fixed[:-3])


def test_bound_accepts_emulated_interpolation_and_rejects_its_faults():
    import numpy as np
    g = np.random.RandomState(8)
    ts, C = 2, 18
    c = np.unique(np.concatenate([g.randint(0, 2, (600, 1)), g.randint(-6, 6, (600, 3)) * ts], 1), axis=0)
    feats = torch.from_numpy(g.randn(c.shape[0], C)).float().bfloat16()
    q = np.concatenate([g.randint(0, 2, (500, 1)), g.randint(-13, 13, (500, 3))], 1)
    ref, A, n_red, rows, wt = B.interp_ref(c, feats, ts, q)
    f = feats.float()
    out = (f[rows.clamp(min=0)] * (rows >= 0)[..., None] * wt.float()[..., None]).sum(1)
    B.assert_within(out, ref, A, n_red, B.OUT_REL_F32, 'emulated interpolation')
    assert bool((rows < 0).any() & (rows >= 0).any()) and bool((np.asarray(q)[:, 1:] < 0).any())
    B.assert_rejects(B.interp_faults(out, c, feats, ts, q), ref, A, n_red, B.OUT_REL_F32)


# ------------------------------------------------------------------------------------------------ fp32 (parity) kernels
def test_bound_accepts_emulated_fp32_simt_conv_and_rejects_its_faults():
    """The fp32 SIMT convolution (64-row tiles, 16-channel reduction chunks) emulated in fp32 passes the bound with the
    fp32 output rounding, and its faults, the dropped last (partial) 16-channel chunk included, are rejected at C_ACC."""
    gen = torch.Generator().manual_seed(9)
    n_in, n_out, K, cin, cout = 400, 300, 27, 40, 70
    nbr = B.random_kernel_map(n_in, n_out, K, gen, empty_offset=5, single_offset=7, empty_tile=1, tile_rows=64)
    for w_layout in (1, 0):
        x = torch.randn(n_in, cin, generator=gen)
        w = torch.randn((K, cin, cout) if w_layout else (K, cout, cin), generator=gen) / (K * cin) ** 0.5
        ref, A, n_red = B.gather_gemm(x, w, nbr, w_layout)
        out = B.gather_gemm(x, w, nbr, w_layout, dtype=torch.float32)[0]
        B.assert_within(out, ref, A, n_red, B.OUT_REL_F32, f'emulated fp32 conv, layout {w_layout}')
        assert bool((out[64:128] == 0).all())
        faults = B.conv_faults(out, x, w, nbr, w_layout, tile_rows=64, chunk=16)
        assert 'reduction channels 32..39' in faults[2][0]
        B.assert_rejects(faults, ref, A, n_red, B.OUT_REL_F32)


def test_bound_rejects_a_dropped_simt_wgrad_split_in_fp32():
    """An fp32-emulated SIMT weight gradient (n_red = pairs + splits) passes the bound; with one pair split of an offset
    missing it is rejected at C_ACC."""
    gen = torch.Generator().manual_seed(10)
    K, n_rows, cin, cout = 27, 3000, 64, 64
    counts = [0, 5] + [int(c) for c in torch.randint(1, n_rows + 1, (K - 2, ), generator=gen)]
    splits = B.simt_wgrad_splits(sum(counts), K, cin, cout, 132)
    assert splits == 6 and B.simt_wgrad_splits(sum(counts), K, 640, 640, 132) == 1
    pin, pout, koff = B.random_pairs(counts, n_rows, n_rows, gen)
    x, dy = torch.randn(n_rows, cin, generator=gen), torch.randn(n_rows, cout, generator=gen)
    ref, A, n_red = B.pair_wgrad(x, dy, pin, pout, koff)
    out = B.pair_wgrad(x, dy, pin, pout, koff, dtype=torch.float32)[0]
    B.assert_within(out, ref, A, n_red + splits, B.OUT_REL_F32, 'emulated fp32 wgrad')
    faults = B.wgrad_faults(out, x, dy, pin, pout, koff, B.simt_wgrad_split_len(max(counts), splits))
    B.assert_rejects(faults, ref, A, n_red + splits, B.OUT_REL_F32)


def test_bound_rejects_a_dropped_direct_wgrad_pixel_slice():
    """The direct fp32 weight gradient on operands in {-1, 0, 1} is exact whatever order its atomics add the pixel slices
    in; the same without its last pixel slice is rejected at C_ACC (n_red = pixels + slices)."""
    gen = torch.Generator().manual_seed(11)
    n, cin, cout, hw = 2, 24, 40, (31, 45)
    M = n * hw[0] * hw[1]
    slice_len, n_slices = B.direct_wgrad_slices(M, cin, cout, 9, 132)
    assert (slice_len, n_slices) == (64, 44)
    assert B.direct_wgrad_slices(M, 3, 16, 49, 132) == (64, 44) and B.direct_wgrad_slices(10 ** 6, 64, 64, 9, 132)[1] == 30
    d = (16.0 / M) ** 0.5
    x, dy = B.ternary((n, cin) + hw, d, gen), B.ternary((n, cout) + hw, d, gen)
    ref, A, n_red = B.dense_wgrad_ref(x, dy, (cout, cin, 3, 3), 1, 1)
    out = torch.nn.grad.conv2d_weight(x, (cout, cin, 3, 3), dy, 1, 1)
    B.assert_exact(out, ref, A, 'emulated direct wgrad', out_bf16=False)
    faults = B.direct_wgrad_slice_faults(out, x, dy, (cout, cin, 3, 3), 1, 1, slice_len)
    assert f'at {(n_slices - 1) * slice_len}' in faults[0][0]
    B.assert_rejects(faults, ref, A, n_red + n_slices, B.OUT_REL_F32)


def test_fp32_norm_bound_accepts_emulated_norm():
    """An fp32 InstanceNorm + ELU emulated in fp32 (torch's rsqrt and expm1) passes the bound with the documented function
    errors as fixed terms (bf16_bounds.seg_norm_fn_fixed); channel 0 with the wrong rstd is rejected."""
    gen = torch.Generator().manual_seed(12)
    sizes, C = [300, 37, 129], 12
    x = torch.randn(sum(sizes), C, generator=gen) * 2 + 0.5
    gamma, beta = torch.rand(C, generator=gen) + 0.5, torch.randn(C, generator=gen)
    z, A, n_red, st = B.seg_norm_ref(x, sizes, gamma, beta, 1e-8)
    seg = st['seg']
    mean = torch.zeros(len(sizes), C).index_add_(0, seg, x) / torch.tensor(sizes, dtype=torch.float32).view(-1, 1)
    d = x - mean[seg]
    var = torch.zeros(len(sizes), C).index_add_(0, seg, d * d) / torch.tensor(sizes, dtype=torch.float32).view(-1, 1)
    y = B._act(d * torch.rsqrt(var + 1e-8)[seg] * gamma + beta, 2)
    F_y = B.seg_norm_fn_fixed(x, gamma, st, z, 2)
    B.assert_within(y, B._act(z, 2), A, n_red, B.OUT_REL_F32, 'emulated fp32 norm', fixed=F_y)
    bad = y.clone()
    bad[:, 0] = B._act(d[:, 0] * torch.rsqrt(var[:, 0] + 1e-4)[seg] * gamma[0] + beta[0], 2)
    B.assert_rejects([('rstd of channel 0 off', bad)], B._act(z, 2), A, n_red, B.OUT_REL_F32, F_y)
