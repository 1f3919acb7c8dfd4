"""CPU: the depth video's split select and the frame dealing of render_video_4k_sharded without a GPU -- the numpy
restatement of k4_op_masked_quantiles_hist / _select (per-share histograms, summed, then selected) against np.percentile
over shares, the argument checks of the two C entry points, and k4nerf.dist.render_video_frames on gloo world 2 and 3
with a stand-in frame renderer (dealing, on_frame order, any dst, arrays equal to the one-process run)."""
import ctypes as C
import os
import socket

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

from k4nerf.utils import (MQ_HIST_LEN, depth_video_frames, depth_video_frames_sharded, masked_quantiles_hist_np,
                          masked_quantiles_select_np)
from test_video import _adversarial, _same

K4_ERR_INVALID_ARG, K4_ERR_WORKSPACE = -1, -4
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _split_select(shares, q):
    """Each pass: every share's histogram, summed, then one select on the sum."""
    state = {}
    for p in range(3):
        hist = sum(masked_quantiles_hist_np(p, s, state) for s in shares)
        assert hist.dtype == np.int64 and hist.shape == (MQ_HIST_LEN,)
        res = masked_quantiles_select_np(p, hist, q, state)
    return res


def _shares(v, k, how):
    if how == 'interleaved':                              # ties and neighbours land on different shares
        return [v[i::k] for i in range(k)]
    if how == 'first_holds_all':                          # every other share empty
        return [v] + [v[:0]] * (k - 1)
    cut = np.sort(np.random.default_rng(k).integers(0, v.size + 1, k - 1))
    return np.split(v, cut)                               # uneven, some possibly empty


@pytest.mark.parametrize('name,v', list(_adversarial()), ids=[n for n, _ in _adversarial()])
@pytest.mark.parametrize('k', [1, 2, 3, 8])
@pytest.mark.parametrize('how', ['interleaved', 'first_holds_all', 'uneven'])
@pytest.mark.parametrize('q', [(5, 95), (0, 100), (50, 33.3)])
def test_split_select_is_np_percentile(name, v, k, how, q):
    """Bit for bit np.percentile over all shares (a zero may differ in sign, as numpy treats -0.0 == 0.0); the NaN case
    has its NaN in one share only."""
    with np.errstate(invalid='ignore'):
        want = np.percentile(v, q=list(q))
    dmin, dmax, count = _split_select(_shares(v, k, how), q)
    assert count == v.size
    for g, w in zip((dmin, dmax), want):
        assert isinstance(g, np.float64) and _same(g, w), (g, w)
        if not (np.isnan(w) or w == 0):
            assert np.float64(g).tobytes() == np.float64(w).tobytes()


def test_split_select_without_values():
    dmin, dmax, count = _split_select([np.zeros(0, np.float32)] * 3, (5, 95))
    assert count == 0 and np.isnan(dmin) and np.isnan(dmax)


def test_split_select_large_ties_across_shares():
    rng = np.random.default_rng(4)
    v = np.concatenate([rng.integers(0, 5, 40000) * 0.5, rng.standard_normal(30000) * 1e-30,
                        np.full(5000, 3e38)]).astype(np.float32)
    rng.shuffle(v)
    for q in ((5, 95), (0, 100), (12.5, 87.5)):
        want = np.percentile(v, q=list(q))
        got = _split_select(_shares(v, 5, 'uneven'), q)
        assert [np.float64(g).tobytes() for g in got[:2]] == [np.float64(w).tobytes() for w in want]


def test_sharded_depth_video_on_one_process_is_depth_video_frames():
    """Without a process group the split path runs on the one share: frames and range as depth_video_frames'."""
    from test_video import _scene
    depths, bgmaps = _scene(n=4, H=7, W=11, seed=5)
    for flipy, rot90 in ((False, 0), (True, 3)):
        want, rw = depth_video_frames(depths, bgmaps, render_video_flipy=flipy, render_video_rot90=rot90, return_range=True)
        got, rg = depth_video_frames_sharded(depths, bgmaps, render_video_flipy=flipy, render_video_rot90=rot90,
                                             return_range=True)
        assert np.array_equal(got, want)
        assert [np.float64(x).tobytes() for x in rg] == [np.float64(x).tobytes() for x in rw]
    with pytest.raises(ValueError):
        depth_video_frames_sharded(depths, np.full_like(bgmaps, 0.5))
    with pytest.raises(ValueError):
        depth_video_frames_sharded(depths, bgmaps, q=(5, 101))


def test_split_entry_points_validate_arguments_without_a_gpu():
    """Bad passes, null pointers, shapes, quantiles and misaligned pointers are K4_ERR_INVALID_ARG, a short workspace
    K4_ERR_WORKSPACE, all before any CUDA call (there is no GPU here); a share without frames launches nothing."""
    from k4nerf import _lib
    lib = _lib.lib
    wsz = lib.k4_op_masked_quantiles_pass_workspace_bytes()
    assert wsz == 256
    header = open(os.path.join(ROOT, 'include', 'k4nerf.h')).read()
    assert '#define K4_MASKED_QUANTILES_HIST_LEN (4 * 2048 + 2)' in header
    assert _lib.K4_MASKED_QUANTILES_HIST_LEN == MQ_HIST_LEN == 4 * 2048 + 2
    buf = C.create_string_buffer(wsz + 64)
    b = (C.addressof(buf) + 15) // 16 * 16
    st = (C.c_int64 * 3)(12 * 10, 10, 1)
    q = (C.c_double * 2)(0.05, 0.95)

    def hist(**kw):
        a = dict(p=0, d=b, g=b, n=2, H=12, W=10, sd=st, sg=st, h=b, ws=b, wsz=wsz)
        a.update(kw)
        return lib.k4_op_masked_quantiles_hist(a['p'], a['d'], a['g'], a['n'], a['H'], a['W'], a['sd'], a['sg'], a['h'],
                                               a['ws'], a['wsz'], None)

    for p in ('d', 'g', 'sd', 'sg', 'h', 'ws'):
        assert hist(**{p: None}) == K4_ERR_INVALID_ARG, p
    for kw in (dict(p=-1), dict(p=3), dict(n=-1), dict(H=0), dict(W=-2), dict(n=0, H=0), dict(n=1 << 20, H=1 << 12),
               dict(ws=b + 8), dict(h=b + 4), dict(d=b + 2), dict(g=b + 1)):
        assert hist(**kw) == K4_ERR_INVALID_ARG, kw
    assert hist(wsz=wsz - 1) == K4_ERR_WORKSPACE
    for p in range(3):                                   # no frames: valid, nothing launched, pointers may be NULL
        assert hist(p=p, n=0, d=None, g=None) == 0

    def select(**kw):
        a = dict(p=0, h=b, q=q, out=b, cnt=b + 16, ws=b, wsz=wsz)
        a.update(kw)
        return lib.k4_op_masked_quantiles_select(a['p'], a['h'], a['q'], a['out'], a['cnt'], a['ws'], a['wsz'], None)

    for p in ('h', 'q', 'out', 'cnt', 'ws'):
        assert select(**{p: None}) == K4_ERR_INVALID_ARG, p
    for kw in (dict(p=-1), dict(p=3), dict(q=(C.c_double * 2)(-0.01, 0.5)), dict(q=(C.c_double * 2)(0.5, 1.01)),
               dict(q=(C.c_double * 2)(float('nan'), 0.5)), dict(ws=b + 8), dict(h=b + 4), dict(out=b + 4),
               dict(cnt=b + 4)):
        assert select(**kw) == K4_ERR_INVALID_ARG, kw
    assert select(wsz=wsz - 1) == K4_ERR_WORKSPACE


# ---------------------------------------------------------------------------------------------
# k4nerf.dist.render_video_frames on gloo with a stand-in frame renderer
# ---------------------------------------------------------------------------------------------
H, W, S = 5, 6, 2          # LR frame, SR scale of the stand-in


def _stand_in(seen):
    """A deterministic 'render' of frame i: u8 SR / LR frames and a depth / bgmap with selected and unselected pixels."""
    def render_into(i, sr_u8, lr_u8, depth, bgmap):
        seen.append(i)
        g = torch.Generator().manual_seed(100 + i)
        sr_u8.copy_(torch.randint(0, 256, sr_u8.shape, generator=g, dtype=torch.uint8))
        lr_u8.copy_(torch.randint(0, 256, lr_u8.shape, generator=g, dtype=torch.uint8))
        depth.copy_(2 + torch.randn(H, W, generator=g))
        bgmap.copy_((torch.rand(H, W, generator=g) * 0.2).round(decimals=2))
    return render_into


def _video(n, rot90, with_on_frame, group=None, dst=0):
    seen, frames = [], []
    k = rot90 % 4
    sr_shape = (S * W, S * H, 3) if k & 1 else (S * H, S * W, 3)
    lr_shape = (W, H, 3) if k & 1 else (H, W, 3)
    on_frame = (lambda i, sr, lr: frames.append((i, sr.clone(), lr.clone()))) if with_on_frame else None
    from k4nerf import dist as kdist
    out = kdist.render_video_frames(_stand_in(seen), n, H, W, sr_shape, lr_shape, torch.device('cpu'),
                                    render_video_flipy=True, render_video_rot90=rot90, on_frame=on_frame, group=group,
                                    dst=dst)
    return out, seen, frames


def _video_worker(rank, world, port, cases, q):
    import sys
    sys.path.insert(0, os.path.join(ROOT, '4k-nerf_b200'))
    sys.path.insert(0, os.path.join(ROOT, 'tests'))
    os.environ['MASTER_ADDR'] = '127.0.0.1'
    os.environ['MASTER_PORT'] = str(port)
    dist.init_process_group('gloo', rank=rank, world_size=world)
    res = []
    try:
        for n, dst, rot90, with_on_frame in cases:
            out, seen, frames = _video(n, rot90, with_on_frame, dst=dst)
            res.append((out, seen, [(i, sr.numpy(), lr.numpy()) for i, sr, lr in frames]))
        q.put((rank, res, None))
    except Exception as e:                                                   # reported, not hung on
        q.put((rank, None, repr(e)))
    dist.destroy_process_group()


@pytest.mark.parametrize('world', [2, 3])
def test_video_frames_dealt_over_gloo_ranks(world):
    cases = [(n, dst, rot90, with_on_frame) for n in (1, 2, 5, 7)
             for dst, rot90, with_on_frame in ((0, 0, False), (world - 1, 1, True), (1, 2, False))]
    ctx = mp.get_context('spawn')
    q = ctx.Queue()
    with socket.socket() as s:
        s.bind(('127.0.0.1', 0))
        port = s.getsockname()[1]
    procs = [ctx.Process(target=_video_worker, args=(r, world, port, cases, q)) for r in range(world)]
    for p in procs:
        p.start()
    try:
        got = dict((r, (res, err)) for r, res, err in (q.get(timeout=300) for _ in range(world)))
    finally:
        for p in procs:
            p.join(timeout=60)
            if p.is_alive():
                p.kill()
    assert all(err is None for _, err in got.values()), got
    for c, (n, dst, rot90, with_on_frame) in enumerate(cases):
        (sr1, lr1, depth1), _, frames1 = _video(n, rot90, with_on_frame)          # one process, no group
        for rank in range(world):
            out, seen, frames = got[rank][0][c]
            assert seen == list(range(rank, n, world)), (c, rank)                 # frame i on rank i % world
            if rank != dst:
                assert out == (None, None, None) and frames == []
                continue
            sr, lr, depth = out
            assert (sr is None) == with_on_frame
            if not with_on_frame:
                assert np.array_equal(sr, sr1)
            assert np.array_equal(lr, lr1) and np.array_equal(depth, depth1), c
            assert [f[0] for f in frames] == [f[0] for f in frames1] == (list(range(n)) if with_on_frame else [])
            for (_, a, b), (_, a1, b1) in zip(frames, frames1):
                assert np.array_equal(a, a1.numpy()) and np.array_equal(b, b1.numpy())
        # the depth video of the one-process run is depth_video_frames' of all frames
        if rot90 == 0:
            seen, d, bg = [], torch.empty(n, H, W), torch.empty(n, H, W)
            render_into = _stand_in(seen)
            for i in range(n):
                render_into(i, torch.empty(S * H, S * W, 3, dtype=torch.uint8), torch.empty(H, W, 3, dtype=torch.uint8),
                            d[i], bg[i])
            assert np.array_equal(depth1, depth_video_frames(d.numpy(), bg.numpy(), render_video_flipy=True))


def test_render_video_frames_rejects_a_dst_outside_the_group():
    from k4nerf import dist as kdist
    with pytest.raises(ValueError):
        kdist.render_video_frames(_stand_in([]), 2, H, W, (S * H, S * W, 3), (H, W, 3), torch.device('cpu'), dst=1)
