"""esb_sum_partial_rows, the fixed-order finisher behind every split sum of the library: out[j] (+)= part[0][j] +
part[1][j] + ... + part[n_parts - 1][j], added left to right with every add rounded to fp32, whatever block shape and tile
depth the host picks for (n_parts, width). The result must equal, bit for bit, a NumPy float32 left-to-right sum; the
operands span 48 binades of both signs, so any reordering, pairing or fused add shows in the last bits."""
import ctypes

import numpy as np
import pytest
import torch

DEV = 'cuda:0'
# the finisher is a C++ entry point of csrc/scratch.cu that the library's callers share; it is not part of the C ABI
SYMBOL = '_Z20esb_sum_partial_rowsPKfixPfiP11CUstream_st'
WIDTHS = [1, 2, 63, 64, 128, 1024, 147456]        # loss sums, norm statistics (S * C), 2 * C, a conv wgrad (K * Cin * Cout)
N_PARTS = [1, 2, 255, 256, 257, 1172, 5000]
# every pair but 147456 x 5000 (2.9 GB of partials; no split sum of the library comes near it)
SHAPES = [(w, n) for w in WIDTHS for n in N_PARTS if w * n <= 1 << 28]
PAD = 37                                          # columns past `width` the call must leave alone


def _finisher():
    from embodiedscan_b200 import _ffi
    fn = getattr(_ffi.lib(), SYMBOL)
    fn.argtypes = [ctypes.c_void_p, ctypes.c_int, ctypes.c_longlong, ctypes.c_void_p, ctypes.c_int, ctypes.c_void_p]
    fn.restype = ctypes.c_int
    return fn


def _mixed(shape, gen):
    """float32 of both signs over 2^-24 .. 2^24, with some +0 and -0."""
    mant = 1 + torch.rand(shape, generator=gen, device=DEV)
    expo = torch.randint(-24, 25, shape, generator=gen, device=DEV).float()
    sign = torch.randint(0, 2, shape, generator=gen, device=DEV).float() * 2 - 1
    v = sign * mant * torch.exp2(expo)
    zero = torch.rand(shape, generator=gen, device=DEV) < 0.01
    return torch.where(zero, sign * 0.0, v).contiguous()


@pytest.mark.gpu
@pytest.mark.parametrize('accumulate', [0, 1])
@pytest.mark.parametrize('width,n_parts', SHAPES)
def test_sum_partial_rows_bit_exact(width, n_parts, accumulate):
    from embodiedscan_b200._ffi import stream
    gen = torch.Generator(device=DEV).manual_seed(width * 7919 + n_parts * 2 + accumulate)
    part = _mixed((n_parts, width), gen)
    out0 = _mixed((width + PAD,), gen)
    out = out0.clone()
    if not accumulate:
        out[:width] = float('nan')                # overwritten, never read
    rc = _finisher()(part.data_ptr(), n_parts, width, out.data_ptr(), accumulate, stream())
    assert rc == 0
    got = out.cpu().numpy()

    p = part.cpu().numpy()
    ref = out0[:width].cpu().numpy().copy() if accumulate else np.zeros(width, np.float32)
    for r in range(n_parts):
        np.add(ref, p[r], out=ref)
    assert np.array_equal(got[:width].view(np.uint32), ref.view(np.uint32)), \
        f'{int((got[:width].view(np.uint32) != ref.view(np.uint32)).sum())} of {width} columns differ'
    assert np.array_equal(got[width:].view(np.uint32), out0[width:].cpu().numpy().view(np.uint32)), \
        'columns past width were written'
