"""Write tests/golden/resize_quarter_ref.pt: cv2.resize(x, None, fx=1/4, fy=1/4) of seeded float32 frames, the
frames run_sr.py:1136 scores LPIPS on, so that the GPU tests need no cv2.

    python tests/golden/make_golden_resize.py

Records cv2.__version__, whether the build uses IPP, and the formula the outputs were matched with
(k4nerf.utils.resize_quarter's docstring): cv2 builds without IPP may compute another one."""
import os
import sys

import cv2
import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.join(ROOT, '4k-nerf_b200'))
from k4nerf.utils import _resize_quarter_np                     # noqa: E402

SIZES = [(3, 3), (3, 9), (7, 3), (4, 5), (6, 6), (9, 8), (12, 13), (14, 15), (37, 50), (62, 75), (131, 170)]


def main():
    cases = []
    for i, (H, W) in enumerate(SIZES):
        x = np.random.default_rng(100 + i).random((H, W, 3), dtype=np.float32)
        want = cv2.resize(x, None, fx=1 / 4, fy=1 / 4)
        assert np.array_equal(want, _resize_quarter_np(x)), (H, W)
        cases.append({'H': H, 'W': W, 'x': torch.from_numpy(x), 'out': torch.from_numpy(np.ascontiguousarray(want))})
    meta = {'cv2': cv2.__version__, 'ipp': bool(cv2.ipp.useIPP()),
            'formula': 'a + (b - a) * t, columns then rows, pair (n-2, n-1) with t = 1 past the edge; '
                       'rows first and pixel n-1 alone when H or W is 3'}
    out = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'resize_quarter_ref.pt')
    torch.save({'meta': meta, 'cases': cases}, out)
    print(out, meta)


if __name__ == '__main__':
    main()
