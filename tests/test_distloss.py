"""CPU: the distortion loss without a GPU -- the C entry points' argument checks, the float64 restatement the GPU tests
hold the kernels to (train_ref64.flatten_eff_distloss) against the pairwise definition and the closed-form gradient,
and the Python wrappers' argument errors."""
import ctypes as C

import pytest
import torch

import train_ref64 as R

K4_ERR_INVALID_ARG, K4_ERR_WORKSPACE = -1, -4


def test_entry_points_validate_arguments_without_a_gpu():
    """Null pointers, counts below 1 and a missing workspace are K4_ERR_INVALID_ARG, a short workspace
    K4_ERR_WORKSPACE, all before any CUDA call (there is no GPU here)."""
    from k4nerf import _lib
    lib = _lib.lib
    assert lib.k4_op_distloss_workspace_bytes(0) == 0 and lib.k4_op_distloss_workspace_bytes(-3) == 0
    assert lib.k4_op_distloss_workspace_bytes(2048) == 16 + 48
    assert lib.k4_op_distloss_workspace_bytes(2049) == 16 + 2 * 48
    buf = C.create_string_buffer(4096 + 16)
    b = (C.addressof(buf) + 15) // 16 * 16           # any aligned address: nothing is dereferenced before the checks
    wsz = lib.k4_op_distloss_workspace_bytes(100)

    def fwd(**kw):
        a = dict(w=b, m=b, rid=b, n=100, iv=0.1, d_iv=None, loss=b, ws=b, wsz=wsz)
        a.update(kw)
        return lib.k4_op_distloss_forward(a['w'], a['m'], a['rid'], a['n'], a['iv'], a['d_iv'], a['loss'], a['ws'], a['wsz'], None)

    def bwd(**kw):
        a = dict(w=b, m=b, rid=b, n=100, iv=0.1, d_iv=None, g=b, div=1, ws=b, wsz=wsz, out=b)
        a.update(kw)
        return lib.k4_op_distloss_backward(a['w'], a['m'], a['rid'], a['n'], a['iv'], a['d_iv'], a['g'], a['div'], a['ws'],
                                           a['wsz'], a['out'], None)

    def seg(**kw):
        a = dict(w=b, s=b, rid=b, n=100, nr=7, wp=b, wt=b, sp=b, st=b, ws=b, wsz=wsz)
        a.update(kw)
        return lib.k4_op_segment_cumsum(a['w'], a['s'], a['rid'], a['n'], a['nr'], a['wp'], a['wt'], a['sp'], a['st'], a['ws'],
                                        a['wsz'], None)

    for f, ptrs, extra in ((fwd, ('w', 'm', 'rid', 'loss', 'ws'), []),
                           (bwd, ('w', 'm', 'rid', 'g', 'ws', 'out'), []),
                           (seg, ('w', 's', 'rid', 'wp', 'wt', 'sp', 'st', 'ws'), [dict(nr=0), dict(nr=-1)])):
        for p in ptrs:
            assert f(**{p: None}) == K4_ERR_INVALID_ARG, (f.__name__, p)
        for kw in [dict(n=0), dict(n=-5), dict(ws=b + 4)] + extra:
            assert f(**kw) == K4_ERR_INVALID_ARG, (f.__name__, kw)
        assert f(wsz=wsz - 1) == K4_ERR_WORKSPACE, f.__name__
        assert f(wsz=0) == K4_ERR_WORKSPACE, f.__name__


# ---------------------------------------------------------------------------------------------------------------------
# the restatement
# ---------------------------------------------------------------------------------------------------------------------
def _random_list(seed, n_rays=40, max_len=9):
    """A ray-sorted list with gaps (rays without samples, ray 0 included when the draw says so), segments of length
    1, and m sorted within each ray; fp64."""
    g = torch.Generator().manual_seed(seed)
    L = torch.randint(0, max_len + 1, (n_rays,), generator=g)
    L[torch.randint(0, n_rays, (5,), generator=g)] = 1
    L[-1] = max(int(L[-1]), 1)
    ray_id = torch.repeat_interleave(torch.arange(n_rays), L)
    w = torch.rand(ray_id.numel(), generator=g, dtype=torch.float64)
    u = torch.rand(ray_id.numel(), generator=g, dtype=torch.float64)
    m = u[torch.argsort(ray_id.double() * 2 + u)]
    return ray_id, w, m


def _pairwise(w, m, interval, ray_id):
    n = int(ray_id.max()) + 1
    same = ray_id[:, None] == ray_id[None, :]
    pair = (w[:, None] * w[None, :] * (m[:, None] - m[None, :]).abs() * same).sum()
    return (pair + interval / 3 * (w * w).sum()) / n


def _closed_form_grad(w, m, interval, ray_id):
    n = int(ray_id.max()) + 1
    same = ray_id[:, None] == ray_id[None, :]
    idx = torch.arange(w.numel())
    before, after = same & (idx[None, :] < idx[:, None]), same & (idx[None, :] > idx[:, None])
    Wl, Wg = (before * w[None, :]).sum(1), (after * w[None, :]).sum(1)
    WMl, WMg = (before * (w * m)[None, :]).sum(1), (after * (w * m)[None, :]).sum(1)
    return (2 * m * (Wl - Wg) + 2 * (WMg - WMl) + 2 / 3 * interval * w) / n


@pytest.mark.parametrize('seed', range(6))
def test_restatement_equals_pairwise_definition_and_closed_form_gradient(seed):
    ray_id, w, m = _random_list(seed)
    counts = torch.bincount(ray_id)
    assert (counts == 1).any() and (counts == 0).any()
    if seed == 0:
        ray_id = ray_id + 3                           # no rays 0..2: the divisor is still max + 1
    interval = 1 / (17 + seed)
    wl = w.clone().requires_grad_(True)
    loss = R.flatten_eff_distloss(wl, m, interval, ray_id)
    loss.backward()
    ref = _pairwise(w, m, interval, ray_id)
    assert abs(float(loss.detach()) - float(ref)) <= 1e-13 * abs(float(ref))
    g = _closed_form_grad(w, m, interval, ray_id)
    assert torch.allclose(wl.grad, g, rtol=1e-12, atol=1e-15)


# ---------------------------------------------------------------------------------------------------------------------
# the Python wrappers
# ---------------------------------------------------------------------------------------------------------------------
def test_wrappers_reject_bad_arguments_without_a_gpu():
    from k4nerf import dcvgo, ub360_utils_cuda
    from k4nerf.torch_efficient_distloss import flatten_eff_distloss
    w = torch.rand(10)
    rid = torch.zeros(10, dtype=torch.int64)
    with pytest.raises(RuntimeError, match='CUDA'):
        flatten_eff_distloss(w, w, 0.1, rid)
    with pytest.raises(RuntimeError, match='CUDA'):
        ub360_utils_cuda.segment_cumsum(w, w, rid)
    with pytest.raises(RuntimeError, match='CUDA'):
        dcvgo.distortion_loss(w, w, 64, rid)
    with pytest.raises(RuntimeError, match='empty'):
        flatten_eff_distloss(w[:0], w[:0], 0.1, rid[:0])
    with pytest.raises(RuntimeError, match='empty'):
        ub360_utils_cuda.segment_cumsum(w[:0], w[:0], rid[:0])
    for bad in ('0.1', None, True, torch.ones(2), torch.ones(1, dtype=torch.bool)):
        with pytest.raises(RuntimeError, match='interval'):
            flatten_eff_distloss(w, w, bad, rid)
    for args in ((w, w.double(), 0.1, rid), (w, w, 0.1, rid.int()), (w, w[:5], 0.1, rid), (w[None], w[None], 0.1, rid[None]),
                 (w.tolist(), w, 0.1, rid)):
        with pytest.raises(RuntimeError):
            flatten_eff_distloss(*args)
