"""CPU: the numpy restatement of k4_png_encode's filter stage and its PNG reader against PNGs written by PIL and cv2,
and the argument checks of the PNG entry points (csrc/k4_png.cu), which return before any CUDA call."""
import ctypes as C
import io

import numpy as np
import pytest

from png_ref import _filters, filter_np, read_png, unfilter_np


def _frames():
    g = np.random.default_rng(0)
    yy, xx = np.mgrid[0:23, 0:37]
    smooth = np.stack([(xx * 7 + yy * 3) % 256, (xx * yy) % 256, (200 - 5 * yy) % 256], -1)
    return {
        'noise': g.integers(0, 256, (17, 29, 3), dtype=np.uint8),
        'smooth': smooth.astype(np.uint8),
        'smooth+noise': np.clip(smooth + g.integers(-3, 4, smooth.shape), 0, 255).astype(np.uint8),
        'constant': np.full((9, 11, 3), 77, np.uint8),
        '1x1': np.array([[[1, 2, 3]]], np.uint8),
        '1x5': g.integers(0, 256, (1, 5, 3), dtype=np.uint8),
        '6x1': g.integers(0, 256, (6, 1, 3), dtype=np.uint8),
    }


@pytest.mark.parametrize('name', list(_frames()))
def test_filter_round_trip(name):
    f = _frames()[name]
    H, W = f.shape[:2]
    s = filter_np(f)
    assert s.shape == (H * (1 + 3 * W),) and np.all(s.reshape(H, -1)[:, 0] < 5)
    assert np.array_equal(unfilter_np(s, H, W), f)


def test_filter_picks_least_abs_sum_lowest_on_tie():
    # row 0 of a constant frame: Sub and Paeth both give [9 9 9 0 ...], the least sum; Sub is the lower type.
    # Row 1: Up, Average... Up gives all zeros, the least sum, and is the lowest type that does
    f = np.full((2, 4, 3), 9, np.uint8)
    s = filter_np(f).reshape(2, -1)
    assert s[0, 0] == 1
    assert s[1, 0] == 2 and not s[1, 1:].any()
    row, prev = np.arange(12, dtype=np.uint8), np.zeros(12, np.uint8)
    sums = np.abs(_filters(row, prev).view(np.int8).astype(int)).sum(1)
    assert int(filter_np(row.reshape(1, 4, 3))[0]) == int(np.argmin(sums))


@pytest.mark.parametrize('name', list(_frames()))
def test_reader_and_unfilter_on_pil_pngs(name):
    from PIL import Image
    f = _frames()[name]
    buf = io.BytesIO()
    Image.fromarray(f).save(buf, format='png')
    H, W, stream, types = read_png(buf.getvalue())
    assert (H, W) == f.shape[:2] and 'IDAT' in types
    assert np.array_equal(unfilter_np(stream, H, W), f)


@pytest.mark.parametrize('name', list(_frames()))
def test_reader_and_unfilter_on_cv2_pngs(name):
    cv2 = pytest.importorskip('cv2')
    f = _frames()[name]
    ok, enc = cv2.imencode('.png', np.ascontiguousarray(f[..., ::-1]))
    assert ok
    H, W, stream, _ = read_png(enc.tobytes())
    assert np.array_equal(unfilter_np(stream, H, W), f)


def _lib():
    from k4nerf import _lib
    return _lib


def test_bound_and_workspace_sizes():
    L = _lib()
    seg = L.K4_PNG_SEG
    for H, W in [(1, 1), (1, 21845), (3024, 4032), (24576, 1)]:
        n = H * (1 + 3 * W)
        assert L.lib.k4_png_encode_bound(H, W) == n + 5 * (-(-n // seg)) + 63
        assert L.lib.k4_png_workspace_bytes(H, W) >= n
    for H, W in [(0, 5), (5, 0), (-1, 3), (1 << 16, 1 << 16)]:
        assert L.lib.k4_png_encode_bound(H, W) == 0 and L.lib.k4_png_workspace_bytes(H, W) == 0


def test_encode_argument_checks():
    """Every rejected call returns K4_ERR_INVALID_ARG (-1) before touching CUDA: the pointers below are never
    dereferenced."""
    L = _lib()
    H, W = 4, 5
    bound, wsb = L.lib.k4_png_encode_bound(H, W), L.lib.k4_png_workspace_bytes(H, W)
    p, ln, ws = C.c_void_p(0x10000), C.c_void_p(0x20000), C.c_void_p(0x30000)

    def enc(rgb=p, h=H, w=W, out=p, cap=bound, d_len=ln, wsp=ws, wsn=wsb):
        return L.lib.k4_png_encode(rgb, h, w, out, cap, d_len, wsp, wsn, None)
    assert enc(rgb=None) == -1
    assert enc(out=None) == -1
    assert enc(d_len=None) == -1
    assert enc(wsp=None) == -1
    assert enc(h=0) == -1 and enc(w=0) == -1 and enc(h=-3) == -1
    assert enc(cap=bound - 1) == -1
    assert enc(wsn=wsb - 1) == -1
    assert enc(wsp=C.c_void_p(0x30010)) == -1          # workspace not 256-byte aligned
    assert enc(d_len=C.c_void_p(0x20004)) == -1        # length not 8-byte aligned
    assert enc(h=1 << 16, w=1 << 16, cap=1 << 40, wsn=1 << 40) == -1    # over one IDAT chunk
