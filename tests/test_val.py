"""CPU: the joint stage's validation scores (csrc/k4_val.cu) without a GPU -- utils.resize_quarter's numpy restatement
against cv2.resize(fx=fy=1/4) and the committed golden, the kernel's evaluation of numpy's pairwise float32 sum against
np.mean(np.square(a - b)) on contiguous arrays and on the reference's movedim views, numpy_visit_order against numpy's
own allocation, and both C entry points' argument checks."""
import ctypes as C
import os

import numpy as np
import pytest
import torch

from k4nerf import _lib
from k4nerf.utils import _resize_quarter_np, numpy_visit_order, resize_quarter, resize_quarter_size, rgb_mse
from val_ref import pairwise_sum, plan, mse_np

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden', 'resize_quarter_ref.pt')


def _frame(H, W, seed, kind='unit'):
    x = np.random.default_rng(seed).random((H, W, 3), dtype=np.float32)
    if kind == 'wide':
        x = (x * 2000 - 1000).astype(np.float32)
    return x


# ---- resize --------------------------------------------------------------------------------------------------------
SIZES = ([(H, W) for H in range(3, 10) for W in range(3, 10)] + [(H, W) for H in range(12, 16) for W in range(16, 20)] +
         [(756 + i, 1008 + j) for i in range(4) for j in range(4)])


@pytest.mark.parametrize('H,W', SIZES)
def test_resize_restatement_is_cv2(H, W):
    cv2 = pytest.importorskip('cv2')
    for kind in ('unit', 'wide'):
        x = _frame(H, W, H * 100 + W, kind)
        want = cv2.resize(x, None, fx=1 / 4, fy=1 / 4)
        assert want.shape == (*resize_quarter_size(H, W), 3)
        assert np.array_equal(resize_quarter(x), want)


def test_resize_restatement_is_cv2_at_4k_and_on_planar_views():
    cv2 = pytest.importorskip('cv2')
    planes = torch.rand(3, 3024, 4032, generator=torch.Generator().manual_seed(1))
    x = planes.movedim(0, -1).numpy()                                 # the reference's rgb_srsave layout
    assert np.array_equal(resize_quarter(x), cv2.resize(x, None, fx=1 / 4, fy=1 / 4))
    c = np.ascontiguousarray(x[1:, 3:])
    assert np.array_equal(resize_quarter(c), cv2.resize(c, None, fx=1 / 4, fy=1 / 4))


def test_resize_golden():
    g = torch.load(GOLDEN, weights_only=False)
    assert g['meta']['ipp'] and g['meta']['cv2'].startswith('4.13')
    for c in g['cases']:
        assert np.array_equal(_resize_quarter_np(c['x'].numpy()), c['out'].numpy()), (c['H'], c['W'])


@pytest.mark.parametrize('H,W', [(1, 1), (2, 9), (9, 2), (1, 4032)])
def test_resize_rejects_what_cv2_rejects(H, W):
    x = np.zeros((H, W, 3), np.float32)
    cv2 = pytest.importorskip('cv2')
    with pytest.raises(cv2.error):
        cv2.resize(x, None, fx=1 / 4, fy=1 / 4)
    with pytest.raises(ValueError):
        resize_quarter(x)


def test_resize_rejects_other_inputs():
    with pytest.raises(ValueError):
        resize_quarter(np.zeros((8, 8, 3), np.float64))
    with pytest.raises(ValueError):
        resize_quarter(np.zeros((8, 8, 4), np.float32))


# ---- MSE -----------------------------------------------------------------------------------------------------------
def _planar(H, W, seed):
    """A [H, W, 3] view of [3, H, W] planes: the reference's rgb_srsave / rgb_srgt_val layout (run_sr.py:768,1131)."""
    g = torch.Generator().manual_seed(seed)
    return torch.rand(1, 3, H, W, generator=g).squeeze().movedim(0, -1).clamp(0, 1).numpy() if H * W > 1 else \
        torch.rand(3, H, W, generator=g).movedim(0, -1).numpy()


@pytest.mark.parametrize('n', list(range(1, 140)) + [255, 256, 257, 1000, 8191, 8192, 8193, 65537, 361_000, 2_290_000])
def test_pairwise_sum_is_numpy(n):
    x = np.random.default_rng(n).random(n, dtype=np.float32)
    assert np.add.reduce(x) == pairwise_sum(x)
    assert plan(n)[1] <= 2                                      # the kernel evaluates unit subtrees two levels deep


def test_unit_subtrees_are_shallow_at_every_frame_size():
    for n in [3 * h * w for h in range(1, 300) for w in (1, 7, 640, 1008, 4032)] + [3 * 65535 * 65535]:
        assert plan(n)[1] <= 2, n


@pytest.mark.parametrize('H,W', [(1, 1), (1, 2), (2, 3), (5, 7), (16, 43), (100, 33), (189, 252), (756, 1008),
                                 (3024, 4032)])
def test_mse_restatement_is_numpy(H, W):
    a, b = _planar(H, W, 1), _planar(H, W, 2)
    for x, y in ((a, b), (np.ascontiguousarray(a), np.ascontiguousarray(b)), (a, np.ascontiguousarray(b)),
                 (np.ascontiguousarray(a), b)):
        want = np.mean(np.square(x - y))
        got = mse_np(x, y)
        assert type(got) is type(want) is np.float32 and got == want
        assert rgb_mse(x, y) == want
    with np.errstate(divide='ignore'):
        assert mse_np(a, a) == 0 and np.isinf(-10. * np.log10(mse_np(a, a)))


def test_mse_division_is_numpys_float64_one():
    """n = 3 H W above 2^24 and not a float32: numpy divides in float64 and rounds once more."""
    H, W = 2897, 2001
    assert int(np.float32(3 * H * W)) != 3 * H * W
    a, b = _planar(H, W, 3), _planar(H, W, 4)
    assert mse_np(a, b) == np.mean(np.square(a - b))


def test_mse_nan_and_inf():
    a, b = _planar(20, 30, 5).copy(), _planar(20, 30, 6)
    a[3, 4, 1] = np.inf
    assert mse_np(a, b) == np.mean(np.square(a - b)) == np.inf
    a[5, 6, 2] = np.nan
    assert np.isnan(mse_np(a, b)) and np.isnan(np.mean(np.square(a - b)))


def _strided(H, W, layout, g):
    base = {'hwc': lambda: torch.rand(H, W, 3, generator=g),
            'chw': lambda: torch.rand(3, H, W, generator=g).movedim(0, -1),
            'whc': lambda: torch.rand(W, H, 3, generator=g).transpose(0, 1),
            'crop': lambda: torch.rand(H + 2, W + 5, 4, generator=g)[1:-1, 2:-3, 1:],
            'bcast': lambda: torch.rand(1, W, 3, generator=g).expand(H, W, 3),
            'cwh': lambda: torch.rand(3, W, H, generator=g).permute(2, 1, 0)}[layout]
    return base().numpy()


LAYOUTS = ['hwc', 'chw', 'whc', 'crop', 'bcast', 'cwh']


@pytest.mark.parametrize('la', LAYOUTS)
@pytest.mark.parametrize('lb', LAYOUTS)
def test_visit_order_is_numpys(la, lb):
    g = torch.Generator().manual_seed(7)
    for H, W in ((5, 7), (1, 9), (6, 1), (40, 61)):
        a, b = _strided(H, W, la, g), _strided(H, W, lb, g)
        d = a - b
        order = numpy_visit_order(a.shape, [s // 4 for s in a.strides], [s // 4 for s in b.strides])
        # the difference's memory order, outermost first (a size-1 axis may sit anywhere)
        want = [ax for ax in sorted(range(3), key=lambda ax: -d.strides[ax]) if d.shape[ax] > 1]
        assert [ax for ax in order if d.shape[ax] > 1] == want, (la, lb, H, W, d.strides)
        assert mse_np(a, b) == np.mean(np.square(d)), (la, lb, H, W)


# ---- the C entry points' argument checks (no CUDA call is reached) ------------------------------------------------
def test_resize_quarter_validates_arguments_without_a_gpu():
    lib = _lib.lib
    buf = C.create_string_buffer(64)
    b = C.addressof(buf)
    st = (C.c_int64 * 3)(24, 3, 1)
    neg = (C.c_int64 * 3)(24, -3, 1)
    for args in ((None, 8, 8, st, b), (b, 8, 8, st, None), (b, 8, 8, None, b), (b, 2, 8, st, b), (b, 8, 2, st, b),
                 (b, 65536, 8, st, b), (b, 8, 0, st, b), (b, 8, 8, neg, b), (b + 2, 8, 8, st, b), (b, 8, 8, st, b + 1)):
        assert lib.k4_op_resize_quarter(*args, None) == -1, args


def test_mse_f32_validates_arguments_without_a_gpu():
    lib = _lib.lib
    buf = C.create_string_buffer(1 << 12)
    b = C.addressof(buf)
    st = (C.c_int64 * 3)(24, 3, 1)
    neg = (C.c_int64 * 3)(-24, 3, 1)
    order = (C.c_int32 * 3)(0, 1, 2)
    ws = lib.k4_op_mse_f32_workspace_bytes(8, 8)
    assert 0 < ws <= 1 << 12
    assert lib.k4_op_mse_f32_workspace_bytes(0, 8) == 0 and lib.k4_op_mse_f32_workspace_bytes(8, 65536) == 0

    def call(**kw):
        a = dict(a=b, b_=b, H=8, W=8, sa=st, sb=st, order=order, out=b, ws=b, n=ws)
        a.update(kw)
        return lib.k4_op_mse_f32(a['a'], a['b_'], a['H'], a['W'], a['sa'], a['sb'], a['order'], a['out'], a['ws'], a['n'],
                                 None)

    for kw in (dict(a=None), dict(b_=None), dict(sa=None), dict(sb=None), dict(order=None), dict(out=None), dict(ws=None),
               dict(H=0), dict(W=-1), dict(H=65536), dict(sa=neg), dict(sb=neg), dict(a=b + 1), dict(b_=b + 2),
               dict(out=b + 3), dict(ws=b + 2), dict(order=(C.c_int32 * 3)(0, 0, 2)), dict(order=(C.c_int32 * 3)(0, 1, 3)),
               dict(order=(C.c_int32 * 3)(-1, 1, 2))):
        assert call(**kw) == -1, kw
    assert call(n=ws - 1) == -4
