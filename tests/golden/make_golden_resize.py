"""Generate tests/golden/resize.npz from ``cv2.resize(frame, (w, h), interpolation=cv2.INTER_LINEAR)``, the call mmcv's
``imresize`` makes for the configs' ``Resize(scale=(480, 480), keep_ratio=False)``, on the seeded frames of
resize_cases.py. It writes only that one fixture:

    python tests/golden/make_golden_resize.py

Stored: the cv2 version, every case's source and target size, and per case and view the SHA-256 of cv2's (h, w, 3)
output (resize_cases.py says why digests).
"""
import os
import sys

import cv2
import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
if HERE not in sys.path:
    sys.path.insert(0, HERE)

from resize_cases import CASES, N_VIEWS, digest, frames  # noqa: E402

if __name__ == '__main__':
    out = {'cv2_version': np.array(cv2.__version__)}
    for name, (_, size) in CASES.items():
        out[f'{name}/sizes'] = np.array(CASES[name], dtype=np.int64)
        out[f'{name}/sha256'] = np.stack([digest(cv2.resize(f, size, interpolation=cv2.INTER_LINEAR))
                                          for f in frames(name, N_VIEWS)])
    path = os.path.join(HERE, 'resize.npz')
    np.savez_compressed(path, **out)
    print(f'wrote {path}: {os.path.getsize(path) / 1024:.1f} KiB, cv2 {cv2.__version__}, '
          f'{len(CASES)} cases x {N_VIEWS} views')
