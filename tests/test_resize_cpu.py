"""CPU: the NumPy restatement of cv2's 8-bit INTER_LINEAR resize (oracle/resize_ref.py) against cv2's own bytes
(tests/golden/resize.npz), and the host side of MultiViewResize and inference_scan's img_scale."""
import inspect
import os
import sys

import numpy as np
import pytest
import torch

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden')
if GOLD not in sys.path:
    sys.path.insert(0, GOLD)

from resize_cases import CASES, HALFWAY, N_VIEWS, digest, frames  # noqa: E402

from oracle import resize_ref as R  # noqa: E402


@pytest.fixture(scope='module')
def gold():
    return dict(np.load(os.path.join(GOLD, 'resize.npz')))


def test_fixture_holds_every_case(gold):
    assert str(gold['cv2_version']).startswith('4.')
    for name, sizes in CASES.items():
        assert np.array_equal(gold[f'{name}/sizes'], np.array(sizes)), name
        assert gold[f'{name}/sha256'].shape == (N_VIEWS, 32), name


@pytest.mark.parametrize('name', list(CASES))
def test_oracle_equals_cv2(gold, name):
    """Every byte of cv2's output, on the first two views and the last one of each case."""
    views = (0, 1, N_VIEWS - 1)
    src = frames(name)[list(views)]
    out = R.resize_linear_u8(src, CASES[name][1])
    assert out.shape[1:] == (CASES[name][1][1], CASES[name][1][0], 3)
    for k, v in enumerate(views):
        assert np.array_equal(digest(out[k]), gold[f'{name}/sha256'][v]), (name, v)


@pytest.mark.parametrize('name', HALFWAY)
def test_halfway_coefficients_round_half_to_even(gold, name):
    """cv2 rounds each coefficient on its own, half to even, so a pair still sums to 2048. Rounding halves up instead
    (pairs summing to 2049) gives other bytes, so the fixture decides the question."""
    (W, H), (w, h) = CASES[name]
    axis = (w, W, True) if w > 100 else (h, H, False)
    scale = 1.0 / (np.float64(axis[0]) / np.float64(axis[1]))
    f = ((np.arange(axis[0]) + 0.5) * scale - 0.5).astype(np.float32)
    t = (f - np.floor(f)) * np.float32(R.COEF_SCALE)
    assert (t - np.floor(t) == 0.5).all(), 'every coefficient of the case must be half-way'
    _, _, c0, c1 = R.linear_taps(*axis)
    assert ((c0 + c1) == R.COEF_SCALE).all()
    src = frames(name, 1)
    half_up = R.resize_linear_u8(src, (w, h), rint=lambda x: np.floor(x + np.float32(0.5)))
    assert not np.array_equal(digest(half_up[0]), gold[f'{name}/sha256'][0])


def test_area_switch_needs_exactly_2x_on_both_axes():
    assert R.is_area_2x(960, 960, 480, 480) and R.is_area_2x(480, 640, 240, 320)
    assert not R.is_area_2x(540, 960, 480, 480) and not R.is_area_2x(960, 480, 480, 480)
    assert not R.is_area_2x(961, 961, 480, 480) and not R.is_area_2x(480, 480, 480, 480)


def _mock_resize(monkeypatch):
    from embodiedscan_b200 import transforms
    calls = []

    def fake(img, size):
        calls.append((tuple(img.shape), tuple(size)))
        return torch.zeros((img.shape[0], 3, size[1], size[0]), dtype=torch.uint8)

    monkeypatch.setattr(transforms, 'resize_multiview', fake)
    return calls


@pytest.mark.parametrize('src_wh,scale,factor', [((640, 480), (480, 480), (0.75, 1.0)),
                                                 ((1280, 1024), (480, 480), (0.375, 0.46875)),
                                                 ((640, 480), 320, (0.5, 2 / 3))])
def test_multiview_resize_meta(monkeypatch, src_wh, scale, factor):
    """The keys mmcv's Resize._resize_img leaves (MultiViewPipeline keeps the last view's): img_shape (h, w),
    scale (w, h), scale_factor (w / W, h / H) as Python floats, keep_ratio."""
    from embodiedscan_b200.registry import TRANSFORMS
    calls = _mock_resize(monkeypatch)
    t = TRANSFORMS.build(dict(type='MultiViewResize', scale=scale, keep_ratio=False))
    W, H = src_wh
    w, h = (scale, scale) if isinstance(scale, int) else scale
    res = t(dict(img=torch.zeros((20, H, W, 3), dtype=torch.uint8), depth_shift=1000.))
    assert calls == [((20, H, W, 3), (w, h))]
    assert res['img'].shape == (20, 3, h, w)
    assert res['img_shape'] == (h, w) and res['scale'] == (w, h) and res['keep_ratio'] is False
    assert res['scale_factor'] == factor and all(type(f) is float for f in res['scale_factor'])
    assert res['depth_shift'] == 1000.


def test_multiview_resize_rejects_modes_it_does_not_build():
    from embodiedscan_b200.transforms import MultiViewResize, resize_multiview
    with pytest.raises(ValueError, match='keep_ratio'):
        MultiViewResize(scale=(480, 480), keep_ratio=True)
    with pytest.raises(ValueError, match='bilinear'):
        MultiViewResize(scale=(480, 480), interpolation='nearest')
    with pytest.raises(AssertionError, match='one source size'):      # frames of several sizes arrive as a list
        resize_multiview([torch.zeros((480, 640, 3), dtype=torch.uint8)] * 2, (480, 480))
    with pytest.raises(AssertionError, match='GPU'):                   # no host fallback
        resize_multiview(torch.zeros((2, 480, 640, 3), dtype=torch.uint8), (480, 480))


def test_inference_scan_keeps_native_size_by_default():
    from embodiedscan_b200.inference import inference_scan
    assert inspect.signature(inference_scan).parameters['img_scale'].default is None
