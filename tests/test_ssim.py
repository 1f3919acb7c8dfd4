"""CPU: the SSIM metric without a GPU -- the numpy path of utils.rgb_ssim against the reference's own rgb_ssim
(tests/golden/make_golden_ssim.py), and the argument checks of the C entry points k4_op_rgb_ssim /
k4_op_rgb_ssim_workspace_bytes."""
import ctypes as C
import os

import numpy as np
import pytest
import torch

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden', 'ssim_ref.pt')
K4_ERR_INVALID_ARG, K4_ERR_WORKSPACE = -1, -4
K4_DTYPE_F32, K4_DTYPE_F64 = 0, 1


def golden_cases():
    return torch.load(GOLD, map_location='cpu', weights_only=False)['cases']


@pytest.mark.parametrize('name', sorted(golden_cases()))
def test_numpy_path_matches_the_reference(name):
    """Every map element within 1e-11 of the reference's scipy-based rgb_ssim, on fp64 pairs; the mean too."""
    from k4nerf.utils import rgb_ssim
    c = golden_cases()[name]
    a, b = c['img0'].numpy(), c['img1'].numpy()
    m = rgb_ssim(a, b, return_map=True, **c['kwargs'])
    assert m.shape == tuple(c['map'].shape)
    assert np.abs(m - c['map'].numpy()).max() <= 1e-11
    assert abs(rgb_ssim(a, b, **c['kwargs']) - c['mean']) <= 1e-11


def test_window_helper_is_the_numpy_paths_window():
    """Both paths take their taps from one helper: normalised, symmetric, centred for odd and even sizes."""
    from k4nerf.utils import _ssim_window
    for f in (1, 8, 11, 31):
        w = _ssim_window(f, 1.5)
        assert w.dtype == np.float64 and w.shape == (f,) and abs(w.sum() - 1) < 1e-15
        assert np.array_equal(w, w[::-1])


def test_entry_points_validate_arguments_without_a_gpu():
    """Null pointers (d_map excepted), filter sizes outside 1..31, images smaller than the window and unknown dtypes are
    K4_ERR_INVALID_ARG, a short workspace K4_ERR_WORKSPACE, all before any CUDA call (there is no GPU here)."""
    from k4nerf import _lib
    lib = _lib.lib
    # one fp64 partial sum per 32 x 32 output tile
    assert lib.k4_op_rgb_ssim_workspace_bytes(11, 11, 11) == 8
    assert lib.k4_op_rgb_ssim_workspace_bytes(756, 1008, 11) == 8 * 24 * 32
    assert lib.k4_op_rgb_ssim_workspace_bytes(3024, 4032, 11) == 8 * 95 * 126
    for H, W, f in ((10, 11, 11), (11, 10, 11), (40, 40, 0), (40, 40, 32), (40, 40, -1), (0, 0, 1)):
        assert lib.k4_op_rgb_ssim_workspace_bytes(H, W, f) == 0, (H, W, f)
    buf = C.create_string_buffer(4096 + 16)
    b = (C.addressof(buf) + 15) // 16 * 16           # any aligned address: nothing is dereferenced before the checks
    st = (C.c_int64 * 3)(3 * 40, 3, 1)
    win = (C.c_double * 31)(*([1.0 / 11] * 31))
    wsz = lib.k4_op_rgb_ssim_workspace_bytes(40, 50, 11)

    def call(**kw):
        a = dict(i0=b, i1=b, dtype=K4_DTYPE_F32, H=40, W=50, s0=st, s1=st, win=win, f=11, map=None, mean=b, ws=b, wsz=wsz)
        a.update(kw)
        return lib.k4_op_rgb_ssim(a['i0'], a['i1'], a['dtype'], a['H'], a['W'], a['s0'], a['s1'], a['win'], a['f'],
                                  1e-4, 9e-4, a['map'], a['mean'], a['ws'], a['wsz'], None)

    for p in ('i0', 'i1', 's0', 's1', 'win', 'mean', 'ws'):
        assert call(**{p: None}) == K4_ERR_INVALID_ARG, p
    for kw in (dict(f=0), dict(f=32), dict(f=-3), dict(H=10), dict(W=10), dict(H=0), dict(dtype=2), dict(dtype=-1),
               dict(ws=b + 4), dict(mean=b + 4), dict(map=b + 4)):
        assert call(**kw) == K4_ERR_INVALID_ARG, kw
    assert call(wsz=wsz - 1) == K4_ERR_WORKSPACE
    assert call(wsz=0) == K4_ERR_WORKSPACE
