"""Cases of tests/golden/resize.npz: source frame sizes and target sizes of ``cv2.resize(..., INTER_LINEAR)``, and the
seeded frames resized.

Frames are uniform random bytes, which do not compress: 50 views of every case would take ~300 MB. The fixture therefore
stores, per case and view, the SHA-256 of cv2's output, and the frames are regenerated here with numpy's legacy
``RandomState``, whose stream NumPy keeps fixed across versions. A digest equal to the stored one is the same output,
byte for byte.
"""
import hashlib

import numpy as np

N_VIEWS = 50          # the largest scan of the configs' test pipeline (MultiViewPipeline n_images=50)

# name: ((W, H) source, (w, h) target)
CASES = {
    'scannet_640x480': ((640, 480), (480, 480)),
    '3rscan_960x540': ((960, 540), (480, 480)),                # exactly 2x on x only: stays linear
    'matterport_1280x1024': ((1280, 1024), (480, 480)),
    'upscale_320x240': ((320, 240), (480, 480)),
    'area_960x960': ((960, 960), (480, 480)),                  # exactly 2x on both axes: cv2 switches to INTER_AREA
    'area_640x480_to_320x240': ((640, 480), (320, 240)),
    'area_y_only_480x960': ((480, 960), (480, 480)),           # exactly 2x on y only: stays linear
    'copy_480x480': ((480, 480), (480, 480)),                  # same size: a copy
    'odd_641x479': ((641, 479), (480, 480)),
    'odd_333x251_to_97x61': ((333, 251), (97, 61)),
    'odd_7x5_to_3x2': ((7, 5), (3, 2)),
    'one_px_wide_1x480': ((1, 480), (480, 480)),
    'one_px_high_640x1': ((640, 1), (480, 480)),
    'one_px_1x1_to_7x5': ((1, 1), (7, 5)),
    'halfway_x_5x3_to_2048x4': ((5, 3), (2048, 4)),            # every column coefficient is k + 1/2 before rounding
    'halfway_y_3x7_to_4x2048': ((3, 7), (4, 2048)),            # every row coefficient is k + 1/2 before rounding
    'upscale_640x480_to_800x600': ((640, 480), (800, 600)),
}
HALFWAY = ('halfway_x_5x3_to_2048x4', 'halfway_y_3x7_to_4x2048')


def frames(name: str, n_views: int = N_VIEWS) -> np.ndarray:
    """(n_views, H, W, 3) uint8: view v of case i is ``RandomState(1000 * i + v)``."""
    (W, H), _ = CASES[name]
    i = list(CASES).index(name)
    return np.stack([np.random.RandomState(1000 * i + v).randint(0, 256, size=(H, W, 3), dtype=np.uint8)
                     for v in range(n_views)])


def digest(frame_hwc: np.ndarray) -> np.ndarray:
    """SHA-256 of one (h, w, 3) uint8 frame in C order, as 32 uint8."""
    assert frame_hwc.dtype == np.uint8 and frame_hwc.ndim == 3
    return np.frombuffer(hashlib.sha256(np.ascontiguousarray(frame_hwc).tobytes()).digest(), dtype=np.uint8)
