"""Generate the golden fixture of the SSIM metric (run where the reference checkout exists, like make_golden_act.py; the
existing fixtures are not regenerated).

    python tests/golden/make_golden_ssim.py

 ssim_ref.pt   the reference's own lib/utils.py rgb_ssim (scipy.signal.convolve2d blur, lib/utils.py:88-134) on fp64
               image pairs, per case: img0, img1 [H, W, 3] float64, the keyword arguments, the map and the mean.
                 fp64_11x11 / fp64_37x53 / fp64_64x80   a noisy pair (a 1x1 map for 11x11)
                 even_window                            filter_size=8 (the half-pixel-shifted taps)
                 params                                 filter_size=7, filter_sigma=2.2, k1=0.02, k2=0.05
                 max255                                 0-255 images with max_val=255
                 identical                              one image against itself (1 everywhere)
                 constant                               a constant image (zero variance) against a noisy one
                 unclamped                              values outside [0, 1], like the unclamped rgb_feature
 The images are fp64 on purpose: the reference forms img**2 in the input's dtype, so fp32 inputs would make it differ from
 utils.rgb_ssim, which works in fp64 throughout.
 lib/utils.py itself imports the reference's CUDA extensions, so only its rgb_ssim definition is loaded, from its file.
"""
import ast
import os

import numpy as np
import scipy.ndimage
import scipy.signal
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
REFERENCE = '/root/reference'


def _reference_rgb_ssim():
    path = os.path.join(REFERENCE, 'lib', 'utils.py')
    tree = ast.parse(open(path).read(), path)
    fn = next(n for n in tree.body if isinstance(n, ast.FunctionDef) and n.name == 'rgb_ssim')
    ns = {'np': np, 'scipy': scipy}
    exec(compile(ast.Module(body=[fn], type_ignores=[]), path, 'exec'), ns)
    return ns['rgb_ssim']


def _pair(rng, h, w, noise=0.1, lo=0.0, hi=1.0):
    a = scipy.ndimage.uniform_filter(rng.uniform(lo, hi, (h, w, 3)), size=(3, 3, 1))      # some local structure
    return a, np.clip(a + noise * (hi - lo) * rng.standard_normal((h, w, 3)), lo, hi)


def cases():
    rng = np.random.default_rng(123)
    out = {}
    for h, w in ((11, 11), (37, 53), (64, 80)):
        out[f'fp64_{h}x{w}'] = (*_pair(rng, h, w), dict(max_val=1))
    out['even_window'] = (*_pair(rng, 29, 41), dict(max_val=1, filter_size=8))
    out['params'] = (*_pair(rng, 30, 26, noise=0.2), dict(max_val=1, filter_size=7, filter_sigma=2.2, k1=0.02, k2=0.05))
    out['max255'] = (*_pair(rng, 33, 47, lo=0.0, hi=255.0), dict(max_val=255))
    a, _ = _pair(rng, 25, 31)
    out['identical'] = (a, a.copy(), dict(max_val=1))
    _, b = _pair(rng, 25, 31)
    out['constant'] = (np.full((25, 31, 3), 0.375), b, dict(max_val=1))
    a = 1.6 * rng.standard_normal((34, 45, 3)) + 0.5
    out['unclamped'] = (a, a + 0.3 * rng.standard_normal((34, 45, 3)), dict(max_val=1))
    return out


def main():
    ref = _reference_rgb_ssim()
    out = {'source': 'reference lib/utils.py rgb_ssim, numpy %s, scipy %s' % (np.__version__, scipy.__version__),
           'cases': {}}
    for name, (a, b, kw) in cases().items():
        m = ref(a, b, return_map=True, **kw)
        out['cases'][name] = {'img0': torch.from_numpy(a.copy()), 'img1': torch.from_numpy(b.copy()), 'kwargs': kw,
                              'map': torch.from_numpy(np.ascontiguousarray(m)), 'mean': float(ref(a, b, **kw))}
        print(name, a.shape, m.shape, out['cases'][name]['mean'])
    torch.save(out, os.path.join(HERE, 'ssim_ref.pt'))


if __name__ == '__main__':
    main()
