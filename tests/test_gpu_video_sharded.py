"""GPU: the depth video's split select and render_video_4k_sharded.  k4_op_masked_quantiles_hist / _select over frames
split into 2, 3 and 8 shares in one process ("virtual ranks", histograms summed with torch) against
k4_op_masked_quantiles over all frames, bit for bit; depth_video_frames_sharded and render_video_4k_sharded on a one-rank
group against the single-GPU functions; two processes sharing the GPU over gloo (tools/video_sharded_check.py), and two
GPUs over NCCL where the box has them."""
import ctypes as C
import json
import os
import socket
import subprocess
import sys

import numpy as np
import pytest
import torch
import torch.distributed as dist

from k4nerf import _lib, render
from k4nerf.utils import depth_video_frames, depth_video_frames_sharded, _strides3

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _stream(dev):
    return C.c_void_p(torch.cuda.current_stream(dev).cuda_stream)


def _fused(d, b, q=(0.05, 0.95)):
    """k4_op_masked_quantiles over all frames: [dmin, dmax, count] as int64 bits."""
    dev = d.device
    n, H, W = d.shape
    ws = torch.empty(_lib.lib.k4_op_masked_quantiles_workspace_bytes(n, H, W), dtype=torch.uint8, device=dev)
    res = torch.empty(3, dtype=torch.int64, device=dev)
    _lib.check(_lib.lib.k4_op_masked_quantiles(C.c_void_p(d.data_ptr()), C.c_void_p(b.data_ptr()), n, H, W, _strides3(d),
                                               _strides3(b), (C.c_double * 2)(*q), C.c_void_p(res.data_ptr()),
                                               C.c_void_p(res.data_ptr() + 16), C.c_void_p(ws.data_ptr()), ws.numel(),
                                               _stream(dev)))
    return res.cpu()


def _split(shares, q=(0.05, 0.95)):
    """The three passes with one histogram and one state per share; the histograms summed with torch."""
    dev = shares[0][0].device
    L = _lib.K4_MASKED_QUANTILES_HIST_LEN
    wsz = _lib.lib.k4_op_masked_quantiles_pass_workspace_bytes()
    ws = [torch.empty(wsz, dtype=torch.uint8, device=dev) for _ in shares]
    res = [torch.full((3,), -7, dtype=torch.int64, device=dev) for _ in shares]
    for p in range(3):
        hists = torch.zeros(len(shares), L, dtype=torch.int64, device=dev)
        for (d, b), h, w in zip(shares, hists, ws):
            n, H, W = d.shape
            _lib.check(_lib.lib.k4_op_masked_quantiles_hist(p, C.c_void_p(d.data_ptr()), C.c_void_p(b.data_ptr()), n, H, W,
                                                            _strides3(d), _strides3(b), C.c_void_p(h.data_ptr()),
                                                            C.c_void_p(w.data_ptr()), wsz, _stream(dev)))
        total = hists.sum(0)
        for w, r in zip(ws, res):
            _lib.check(_lib.lib.k4_op_masked_quantiles_select(p, C.c_void_p(total.data_ptr()), (C.c_double * 2)(*q),
                                                              C.c_void_p(r.data_ptr()), C.c_void_p(r.data_ptr() + 16),
                                                              C.c_void_p(w.data_ptr()), wsz, _stream(dev)))
    return [r.cpu() for r in res]


def _shares(d, b, k, empty_first=False):
    """Frames dealt round-robin (frame i to share i % k, as render_video_4k_sharded deals them); with ``empty_first``
    the first share gets none."""
    if empty_first:
        return [(d[:0], b[:0])] + _shares(d, b, k - 1)
    return [(d[i::k], b[i::k]) for i in range(k)]


def _frames(n, H, W, seed, sel=0.6, levels=None):
    g = torch.Generator().manual_seed(seed)
    d = 2 + torch.randn(n, H, W, generator=g)
    if levels:
        d = torch.round(d * levels) / levels
    bg = (torch.rand(n, H, W, generator=g) * (0.1 / sel)).clamp(0, 1)
    return d.float(), bg.float()


def _edge_cases():
    yield 'one_value', torch.tensor([[[3.5]]]), torch.zeros(1, 1, 1)
    yield 'ties', *_frames(7, 9, 13, 1, levels=2)
    yield 'one_level', torch.full((5, 4, 6), 0.25), torch.zeros(5, 4, 6)
    d, b = _frames(6, 8, 10, 2)
    b[1::2] = 0.5                                                       # every other frame selects nothing
    yield 'none_in_some_shares', d, b
    d, b = _frames(6, 8, 10, 3)
    d[4, 2, 3], b[4, 2, 3] = float('nan'), 0.0                          # a NaN in one share
    yield 'nan_in_one_share', d, b
    d, b = _frames(5, 8, 10, 4)
    b[:] = 0.5                                                          # nothing selected anywhere
    yield 'none_selected', d, b
    d, b = _frames(4, 6, 7, 5)
    d[0, 0, :4] = torch.tensor([float('inf'), -float('inf'), 0.0, -0.0])
    b[0, 0, :4] = 0.0
    yield 'inf_and_zeros', d, b


@pytest.mark.parametrize('case', list(_edge_cases()), ids=[c[0] for c in _edge_cases()])
@pytest.mark.parametrize('k', [2, 3, 8])
def test_split_passes_are_the_fused_op(cuda_device, case, k):
    _, d, b = case
    d, b = d.to(cuda_device), b.to(cuda_device)
    for empty_first in (False, True):
        for q in ((0.05, 0.95), (0.0, 1.0)):
            want = _fused(d, b, q)
            for got in _split(_shares(d, b, k, empty_first), q):
                assert torch.equal(got, want), (got, want)                  # every share: the same bits


def test_split_passes_at_120_4k_lr_frames(cuda_device):
    """120 x 756 x 1008 (the LR frames of a 4K video), with ties, and views with the frame axis last."""
    d, b = _frames(120, 756, 1008, 9, levels=64)
    d, b = d.to(cuda_device), b.to(cuda_device)
    want = _fused(d, b)
    assert want[2] > 0
    for k in (2, 3, 8):
        for got in _split(_shares(d, b, k)):
            assert torch.equal(got, want), k
    dv, bv = d.permute(1, 2, 0).contiguous().permute(2, 0, 1), b.permute(1, 2, 0).contiguous().permute(2, 0, 1)
    for got in _split(_shares(dv, bv, 3)):
        assert torch.equal(got, want)


def test_split_passes_do_not_sync_the_host(cuda_device):
    d, b = _frames(8, 64, 96, 11)
    d, b = d.to(cuda_device), b.to(cuda_device)
    _split(_shares(d, b, 3))
    torch.cuda.set_sync_debug_mode('error')
    try:
        shares = _shares(d, b, 3)
        L = _lib.K4_MASKED_QUANTILES_HIST_LEN
        wsz = _lib.lib.k4_op_masked_quantiles_pass_workspace_bytes()
        ws = torch.empty(wsz, dtype=torch.uint8, device=cuda_device)
        res = torch.empty(3, dtype=torch.int64, device=cuda_device)
        h = torch.zeros(L, dtype=torch.int64, device=cuda_device)
        for p in range(3):
            h.zero_()
            for sd, sb in shares:
                _lib.check(_lib.lib.k4_op_masked_quantiles_hist(p, C.c_void_p(sd.data_ptr()), C.c_void_p(sb.data_ptr()),
                                                                *sd.shape, _strides3(sd), _strides3(sb), C.c_void_p(h.data_ptr()),
                                                                C.c_void_p(ws.data_ptr()), wsz, _stream(cuda_device)))
            _lib.check(_lib.lib.k4_op_masked_quantiles_select(p, C.c_void_p(h.data_ptr()), (C.c_double * 2)(0.05, 0.95),
                                                              C.c_void_p(res.data_ptr()), C.c_void_p(res.data_ptr() + 16),
                                                              C.c_void_p(ws.data_ptr()), wsz, _stream(cuda_device)))
    finally:
        torch.cuda.set_sync_debug_mode(0)
    assert torch.equal(res.cpu(), _fused(d, b))


@pytest.fixture
def one_rank_group():
    with socket.socket() as s:
        s.bind(('127.0.0.1', 0))
        port = s.getsockname()[1]
    dist.init_process_group('gloo', init_method=f'tcp://127.0.0.1:{port}', rank=0, world_size=1)
    try:
        yield dist.group.WORLD
    finally:
        dist.destroy_process_group()


def test_depth_video_frames_sharded_on_one_rank(cuda_device, one_rank_group):
    d, b = _frames(5, 30, 41, 13, levels=8)
    d, b = d.to(cuda_device), b.to(cuda_device)
    for flipy, rot90 in ((False, 0), (True, 1), (False, -2)):
        want, rw = depth_video_frames(d, b, render_video_flipy=flipy, render_video_rot90=rot90, return_range=True)
        got, rg = depth_video_frames_sharded(d, b, render_video_flipy=flipy, render_video_rot90=rot90,
                                             group=one_rank_group, return_range=True)
        assert got.is_cuda and torch.equal(got, want)
        assert [np.float64(x).tobytes() for x in rg] == [np.float64(x).tobytes() for x in rw]
    with pytest.raises(ValueError):
        depth_video_frames_sharded(d, torch.full_like(b, 0.5), group=one_rank_group)


def test_render_video_4k_sharded_on_one_rank(cuda_device, one_rank_group):
    from test_gpu_video import H, W, N, _net
    from helpers import make_state, model_from_state
    from oracle import scenes
    m = model_from_state(make_state('cfgA', res=32, regime='shell'), cuda_device)
    m.mlp_mode = 'fp32'
    poses, Ks = [], []
    for th in (30.0, 75.0, 120.0):
        K, c2w = scenes.blender_camera(H, W, theta=th)
        poses.append(c2w.numpy()); Ks.append(K)
    args = (m, _net(cuda_device, 4, 1), np.array(poses), np.array([[H, W]] * N), np.array(Ks), False,
            dict(scenes.RENDER_KW_DVGO))
    for extra in ({}, dict(render_video_flipy=True, render_video_rot90=3)):
        want = render.render_video_4k(*args, test_tile=16, **extra)
        got = render.render_video_4k_sharded(*args, test_tile=16, group=one_rank_group, **extra)
        assert all(np.array_equal(g, w) for g, w in zip(got, want))
    seen = []
    sr, lr, depth = render.render_video_4k_sharded(*args, test_tile=16, on_frame=lambda i, s, l: seen.append(i),
                                                   group=one_rank_group)
    assert sr is None and seen == list(range(N))
    with pytest.raises(ValueError):
        render.render_video_4k_sharded(*args, test_tile=16, group=one_rank_group, dst=1)


def _free_port():
    with socket.socket() as s:
        s.bind(('127.0.0.1', 0))
        return s.getsockname()[1]


def _check(nproc, *flags):
    cmd = [sys.executable, '-m', 'torch.distributed.run', '--nnodes=1', '--nproc-per-node', str(nproc), '--master-addr',
           '127.0.0.1', '--master-port', str(_free_port()), os.path.join(ROOT, 'tools', 'video_sharded_check.py'), *flags]
    p = subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.PIPE, text=True, start_new_session=True)
    try:
        out, err = p.communicate(timeout=900)
    finally:
        if p.poll() is None:                             # a hung run is killed with its workers, not left behind
            os.killpg(p.pid, 9)
            p.wait()
    assert p.returncode == 0, err[-3000:]
    res = json.loads([l for l in out.splitlines() if l.startswith('{')][-1])
    assert res['world'] == nproc and len(res['cases']) == 15
    assert all(c['identical'] for c in res['cases']), [c for c in res['cases'] if not c['identical']]
    return res


def test_two_processes_sharing_the_gpu_over_gloo(cuda_device):
    _check(2, '--backend', 'gloo', '--same-gpu')


@pytest.mark.skipif(not torch.cuda.is_available() or torch.cuda.device_count() < 2, reason='needs 2 GPUs')
def test_two_gpus_over_nccl():
    _check(2, '--backend', 'nccl')
