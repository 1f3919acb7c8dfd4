"""CPU: the depth video of run_sr.py --render_video without a GPU -- the numpy restatement of its percentiles against
np.percentile, the rainbow table against its formulas (and matplotlib where installed), utils.depth_video_frames'
numpy path against a literal transcription of run_sr.py:1459-1463, and the argument checks of the C entry points
k4_op_masked_quantiles / k4_op_depth_video_u8 / k4_op_frame_u8."""
import ctypes as C

import numpy as np
import pytest

from k4nerf.utils import depth_video_frames, masked_quantiles_np, rainbow_lut_u8, to8b

K4_ERR_INVALID_ARG, K4_ERR_WORKSPACE = -1, -4


def _same(a, b):
    """Equal as numpy compares (-0.0 == 0.0), NaN where NaN."""
    a, b = np.float64(a), np.float64(b)
    return (np.isnan(a) and np.isnan(b)) or a == b


def _adversarial():
    rng = np.random.default_rng(0)
    yield 'one', np.array([3.5], np.float32)
    yield 'two', np.array([2.0, -1.0], np.float32)
    yield 'three', np.array([7.0, 7.0, -3.0], np.float32)
    yield 'ties', rng.integers(0, 4, 1001).astype(np.float32)
    yield 'one_value', np.full(777, 0.25, np.float32)
    yield 'negative', (-np.abs(rng.standard_normal(513)) * 1e3).astype(np.float32)
    yield 'signed_zeros', np.array([0.0, -0.0, 0.0, -0.0, 1.0, -1.0, -0.0], np.float32)
    yield 'mixed', np.concatenate([rng.standard_normal(300), np.full(200, -2.0), np.zeros(50), -np.zeros(50)]).astype(np.float32)
    yield 'tiny_range', (1 + rng.integers(0, 3, 999) * np.finfo(np.float32).eps).astype(np.float32)
    yield 'inf', np.array([1.0, np.inf, -np.inf, 2.0], np.float32)
    yield 'nan', np.array([1.0, np.nan, 2.0], np.float32)


@pytest.mark.parametrize('name,v', list(_adversarial()), ids=[n for n, _ in _adversarial()])
@pytest.mark.parametrize('q', [(0, 100), (5, 95), (95, 5), (0, 5), (100, 100), (50, 33.3)])
def test_quantile_restatement_is_np_percentile(name, v, q):
    """Bit for bit np.percentile's values (numpy treats -0.0 and +0.0 as equal, so a zero may differ in sign), both
    np.float64; the shuffled input gives the same values."""
    with np.errstate(invalid='ignore'):
        want = np.percentile(v, q=list(q))
    got = masked_quantiles_np(v, q)
    assert all(isinstance(g, np.float64) for g in got)
    for g, w in zip(got, want):
        assert _same(g, w), (g, w)
        if not (np.isnan(w) or w == 0):
            assert np.float64(g).tobytes() == np.float64(w).tobytes()
    again = masked_quantiles_np(np.random.default_rng(1).permutation(v), q)
    assert all(np.float64(a).tobytes() == np.float64(b).tobytes() for a, b in zip(got, again))


def test_quantile_restatement_errors():
    with pytest.raises(ValueError):
        masked_quantiles_np(np.zeros(0, np.float32))
    for q in ((-1, 5), (5, 101), (5,), (1, 2, 3), (np.nan, 5)):
        with pytest.raises(ValueError):
            masked_quantiles_np(np.ones(4, np.float32), q)


def test_rainbow_table():
    lut = rainbow_lut_u8()
    assert lut.dtype == np.uint8 and lut.shape == (256, 3)
    assert tuple(lut[0]) == (127, 0, 255) and tuple(lut[255]) == (255, 0, 0)
    x = np.arange(256) / 255.0
    want = np.stack([np.abs(2 * x - 0.5), np.sin(np.pi * x), np.cos(np.pi * x / 2)], -1)
    # the formulas up to the last bits of x: an entry may only move by one where 255 * value is within 1e-9 of an integer
    diff = np.abs(lut.astype(int) - np.floor(255 * np.clip(want, 0, 1)).astype(int))
    assert diff.max() <= 1
    assert np.all(np.abs(255 * np.clip(want, 0, 1)[diff > 0] - np.round(255 * np.clip(want, 0, 1)[diff > 0])) < 1e-9)
    assert tuple(lut[64]) == (0, 180, 235)      # x = 64 / 255: 255 |2x - 0.5| = 0.5, 255 sin(pi x) = 180.6, 255 cos(pi x / 2) = 235.4


def test_rainbow_table_is_matplotlibs():
    plt = pytest.importorskip('matplotlib.pyplot')
    cmap = plt.get_cmap('rainbow')
    assert cmap.N == 256
    assert np.array_equal(rainbow_lut_u8(), to8b(cmap(np.arange(256) / 256 + 1e-6)[:, :3]))


def _float_rainbow():
    x = np.linspace(0, 1, 256)
    lut = np.ones((256 + 3, 4))
    lut[:256, 0] = np.clip(np.abs(2 * x - 0.5), 0, 1)
    lut[:256, 1] = np.clip(np.sin(x * np.pi), 0, 1)
    lut[:256, 2] = np.clip(np.cos(x * np.pi / 2), 0, 1)
    lut[256 + 2] = 0.0                                     # set_bad's default, (0, 0, 0, 0)
    return lut


def _get_cmap_rainbow(X):
    """matplotlib's Colormap.__call__(X) for float X, with the rainbow table (N = 256)."""
    N = 256
    xa = np.array(X, copy=True)
    xa *= N
    xa[xa == N] = N - 1
    mask_under, mask_over, mask_bad = xa < 0, xa >= N, np.isnan(xa)
    with np.errstate(invalid='ignore'):
        xa = xa.astype(int)
    xa[mask_under] = N
    xa[mask_over] = N + 1
    xa[mask_bad] = N + 2
    return _float_rainbow().take(xa, axis=0, mode='clip')


def _literal(depths, bgmaps, flipy, rot90):
    """run_sr.py:1459-1463 with render.py's _post flip / rotation of depths and bgmaps before it."""
    depths = [np.rot90(np.flip(d, axis=0) if flipy else d, k=rot90, axes=(0, 1)) for d in depths]
    bgmaps = [np.rot90(np.flip(b, axis=0) if flipy else b, k=rot90, axes=(0, 1)) for b in bgmaps]
    depths, bgmaps = np.array(depths), np.array(bgmaps)
    depths_vis = depths * (1-bgmaps) + bgmaps
    dmin, dmax = np.percentile(depths_vis[bgmaps < 0.1], q=[5, 95])
    with np.errstate(divide='ignore', invalid='ignore'):
        depth_vis = _get_cmap_rainbow(1 - np.clip((depths_vis - dmin) / (dmax - dmin), 0, 1)).squeeze()[..., :3]
    return to8b(depth_vis), (dmin, dmax)


def _scene(n=3, H=9, W=13, seed=0):
    rng = np.random.default_rng(seed)
    depths = (2 + rng.standard_normal((n, H, W, 1))).astype(np.float32)
    bgmaps = np.clip(rng.uniform(-0.2, 0.5, (n, H, W, 1)), 0, 1).astype(np.float32)
    bgmaps[0, 0, 0, 0] = np.float32(0.1)                   # exactly the threshold: not selected
    return depths, bgmaps


@pytest.mark.parametrize('flipy', [False, True])
@pytest.mark.parametrize('rot90', [-1, 0, 1, 2, 3, 4, 5])
def test_numpy_path_is_run_sr_literally(flipy, rot90):
    depths, bgmaps = _scene()
    want, rng_want = _literal(depths, bgmaps, flipy, rot90)
    got, rng_got = depth_video_frames(depths, bgmaps, render_video_flipy=flipy, render_video_rot90=rot90, return_range=True)
    assert got.dtype == np.uint8 and got.shape == want.shape and got.flags['C_CONTIGUOUS']
    assert np.array_equal(got, want)
    assert all(np.float64(g).tobytes() == np.float64(w).tobytes() for g, w in zip(rng_got, rng_want))
    # [n, H, W] frames give the same
    assert np.array_equal(depth_video_frames(depths[..., 0], bgmaps[..., 0], render_video_flipy=flipy,
                                             render_video_rot90=rot90), want)


def test_numpy_path_edge_values():
    """Pixels on dmin and dmax, dmax == dmin (inf and NaN normalisations: colours 255, 0 and 'bad'), a NaN depth."""
    depths, bgmaps = _scene(n=2, H=6, W=7, seed=3)
    depths[1, 2, 3, 0] = np.nan
    bgmaps[1, 2, 3, 0] = 0.5
    want, (dmin, dmax) = _literal(depths, bgmaps, False, 0)
    assert np.array_equal(depth_video_frames(depths, bgmaps), want)
    assert tuple(want[1, 2, 3]) == (0, 0, 0)
    # a constant selected depth: dmax == dmin; unselected pixels above / below / on it
    depths = np.full((2, 5, 6, 1), 1.5, np.float32)
    bgmaps = np.zeros((2, 5, 6, 1), np.float32)
    bgmaps[0, 0, :3, 0] = (0.5, 0.6, 1.0)                  # depths_vis 1.25, 1.3, 1.0: below the range
    depths[1, 1, :2, 0] = (9.0, 1.5)
    bgmaps[1, 1, :2, 0] = (0.2, 0.2)                        # depths_vis 7.4: above; 1.4: below
    want, (dmin, dmax) = _literal(depths, bgmaps, False, 0)
    assert dmin == dmax == 1.5
    got = depth_video_frames(depths, bgmaps)
    assert np.array_equal(got, want)
    assert tuple(got[0, 1, 1]) == (0, 0, 0)                   # 0 / 0: bad
    assert tuple(got[0, 0, 0]) == tuple(rainbow_lut_u8()[255])  # -inf -> x = 1
    assert tuple(got[1, 1, 0]) == tuple(rainbow_lut_u8()[0])    # +inf -> x = 0


def test_numpy_path_errors():
    depths, bgmaps = _scene()
    with pytest.raises(ValueError):
        depth_video_frames(depths, np.full_like(bgmaps, 0.5))          # nothing selected
    with pytest.raises(ValueError):
        depth_video_frames(depths, bgmaps[:, :-1])
    with pytest.raises(ValueError):
        depth_video_frames(depths[0, ..., 0], bgmaps[0, ..., 0])


def test_entry_points_validate_arguments_without_a_gpu():
    """Null pointers, bad shapes, quantiles outside [0, 1], bad flips and misaligned pointers are K4_ERR_INVALID_ARG,
    a short workspace K4_ERR_WORKSPACE, all before any CUDA call (there is no GPU here)."""
    from k4nerf import _lib
    lib = _lib.lib
    wsz = lib.k4_op_masked_quantiles_workspace_bytes(120, 756, 1008)
    assert wsz == 256 + 8 * 4 * 2048
    assert lib.k4_op_masked_quantiles_workspace_bytes(1, 1, 1) == wsz
    for shape in ((0, 4, 4), (4, 0, 4), (4, 4, 0), (-1, 4, 4), (1 << 20, 1 << 12, 1)):
        assert lib.k4_op_masked_quantiles_workspace_bytes(*shape) == 0, shape
    buf = C.create_string_buffer(wsz + 64)
    b = (C.addressof(buf) + 15) // 16 * 16
    st = (C.c_int64 * 3)(12 * 10, 10, 1)
    q = (C.c_double * 2)(0.05, 0.95)

    def quant(**kw):
        a = dict(d=b, g=b, n=2, H=12, W=10, sd=st, sg=st, q=q, out=b, cnt=b + 16, ws=b, wsz=wsz)
        a.update(kw)
        return lib.k4_op_masked_quantiles(a['d'], a['g'], a['n'], a['H'], a['W'], a['sd'], a['sg'], a['q'], a['out'],
                                          a['cnt'], a['ws'], a['wsz'], None)

    for p in ('d', 'g', 'sd', 'sg', 'q', 'out', 'cnt', 'ws'):
        assert quant(**{p: None}) == K4_ERR_INVALID_ARG, p
    for kw in (dict(n=0), dict(H=0), dict(W=-2), dict(n=1 << 20, H=1 << 12), dict(q=(C.c_double * 2)(-0.01, 0.5)),
               dict(q=(C.c_double * 2)(0.5, 1.01)), dict(q=(C.c_double * 2)(float('nan'), 0.5)), dict(ws=b + 8),
               dict(out=b + 4), dict(cnt=b + 4), dict(d=b + 2), dict(g=b + 1)):
        assert quant(**kw) == K4_ERR_INVALID_ARG, kw
    assert quant(wsz=wsz - 1) == K4_ERR_WORKSPACE
    lut = (C.c_uint8 * 768)()

    def video(**kw):
        a = dict(d=b, g=b, n=2, H=12, W=10, sd=st, sg=st, r=b, lut=lut, flip=0, k=0, out=b)
        a.update(kw)
        return lib.k4_op_depth_video_u8(a['d'], a['g'], a['n'], a['H'], a['W'], a['sd'], a['sg'], a['r'], a['lut'],
                                        a['flip'], a['k'], a['out'], None)

    for p in ('d', 'g', 'sd', 'sg', 'r', 'lut', 'out'):
        assert video(**{p: None}) == K4_ERR_INVALID_ARG, p
    for kw in (dict(n=0), dict(H=0), dict(W=0), dict(n=65536), dict(H=65536), dict(W=70000), dict(flip=2),
               dict(flip=-1), dict(r=b + 4), dict(d=b + 2)):
        assert video(**kw) == K4_ERR_INVALID_ARG, kw
    st3 = (C.c_int64 * 3)(30, 3, 1)

    def frame(**kw):
        a = dict(x=b, H=12, W=10, s=st3, flip=0, k=0, out=b)
        a.update(kw)
        return lib.k4_op_frame_u8(a['x'], a['H'], a['W'], a['s'], a['flip'], a['k'], a['out'], None)

    for p in ('x', 's', 'out'):
        assert frame(**{p: None}) == K4_ERR_INVALID_ARG, p
    for kw in (dict(H=0), dict(W=-1), dict(H=65536), dict(flip=3), dict(x=b + 1)):
        assert frame(**kw) == K4_ERR_INVALID_ARG, kw
