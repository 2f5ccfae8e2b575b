"""Oracle (test infrastructure): ``cv2.resize(img, (w, h), interpolation=cv2.INTER_LINEAR)`` on 8-bit frames, in NumPy.

This is the arithmetic behind the configs' ``Resize(scale=(480, 480), keep_ratio=False)`` (mmcv ``imresize`` with its
default cv2 backend and ``'bilinear'``). It restates OpenCV's ``resize`` for CV_8U (imgproc/src/resize.cpp), which works
in fixed point:

  * one coefficient table per axis. For output index d with ``scale = 1 / (out / in)`` in double:
    ``f = float((d + 0.5) * scale - 0.5)``, ``s = floor(f)``, ``f -= s``, and the two coefficients are
    ``rint((1 - f) * 2048)`` and ``rint(f * 2048)`` in float32, each rounded on its own, half to even;
  * columns: a tap left of the source (s < 0) or on or right of its last pixel (s >= in - 1) becomes
    ``s = clamp, f = 0``. Rows keep their coefficients, and only the two row indices are clamped into the source;
  * horizontal pass ``S = p0 * c0 + p1 * c1`` (int32), vertical pass
    ``out = (((b0 * (S0 >> 4)) >> 16) + ((b1 * (S1 >> 4)) >> 16) + 2) >> 2``;
  * an exact 2x downscale on both axes is computed as ``INTER_AREA``: the rounded mean ``(a + b + c + d + 2) >> 2`` of
    each 2x2 block;
  * an unchanged size is a copy.

PINNED by ``tests/golden/resize.npz`` (cv2 itself on seeded frames, ``tests/test_resize_cpu.py``).
"""
import numpy as np

COEF_SCALE = 2048                    # INTER_RESIZE_COEF_SCALE, 11 fractional bits


def linear_taps(n_out: int, n_in: int, clamp_coef: bool, rint=np.rint):
    """cv2's table for one axis: ``(i0, i1, c0, c1)`` int64 arrays of length n_out (source indices already clamped).
    `rint` rounds the scaled float32 coefficients (cv2: half to even); tests pass others to show the fixture tells
    them apart."""
    scale = 1.0 / (np.float64(n_out) / np.float64(n_in))
    f = ((np.arange(n_out, dtype=np.float64) + 0.5) * scale - 0.5).astype(np.float32)
    s = np.floor(f).astype(np.int64)
    f = f - s.astype(np.float32)
    if clamp_coef:
        out_of_range = (s < 0) | (s >= n_in - 1)
        f[out_of_range] = 0
        s = np.clip(s, 0, n_in - 1)
    c0 = rint((np.float32(1) - f) * np.float32(COEF_SCALE)).astype(np.int64)
    c1 = rint(f * np.float32(COEF_SCALE)).astype(np.int64)
    return np.clip(s, 0, n_in - 1), np.clip(s + 1, 0, n_in - 1), c0, c1


def is_area_2x(H: int, W: int, h: int, w: int) -> bool:
    """cv2 switches INTER_LINEAR to INTER_AREA when both scales are exactly the integer 2."""
    sx, sy = 1.0 / (w / W), 1.0 / (h / H)
    return abs(sx - round(sx)) < np.finfo(np.float64).eps and abs(sy - round(sy)) < np.finfo(np.float64).eps and \
        round(sx) == 2 and round(sy) == 2


def resize_linear_u8(img: np.ndarray, size, rint=np.rint) -> np.ndarray:
    """img (..., H, W, C) uint8 -> (..., h, w, C) uint8 for ``size = (w, h)``, bit for bit as cv2.INTER_LINEAR."""
    w, h = size
    H, W = img.shape[-3:-1]
    if (h, w) == (H, W):
        return img.copy()
    x = img.astype(np.int64)
    if is_area_2x(H, W, h, w):
        s = x[..., 0::2, 0::2, :] + x[..., 0::2, 1::2, :] + x[..., 1::2, 0::2, :] + x[..., 1::2, 1::2, :]
        return ((s + 2) >> 2).astype(np.uint8)
    xi0, xi1, a0, a1 = linear_taps(w, W, True, rint)
    yi0, yi1, b0, b1 = linear_taps(h, H, False, rint)
    a0, a1 = a0[:, None], a1[:, None]
    S0 = x[..., yi0, :, :][..., xi0, :] * a0 + x[..., yi0, :, :][..., xi1, :] * a1
    S1 = x[..., yi1, :, :][..., xi0, :] * a0 + x[..., yi1, :, :][..., xi1, :] * a1
    out = (((b0[:, None, None] * (S0 >> 4)) >> 16) + ((b1[:, None, None] * (S1 >> 4)) >> 16) + 2) >> 2
    return out.astype(np.uint8)
