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
