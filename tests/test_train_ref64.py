"""CPU: pin the float64 training-forward restatement (train_ref64.py) that the GPU gradient tests compare the library
with.  (i) Its forward against the oracle pipeline on the CPU ops: identical sample lists, per-ray outputs equal to
fp32 rounding.  (ii) Its gradients against central differences in fp64, on grid entries at corners, faces and the
interior of the grids and on rgbnet weights, for each model kind; every difference step is checked to leave the
sample lists unchanged (no step crosses a threshold)."""
import time

import pytest
import torch

import mpi_act
import train_ref64 as R
from helpers import make_state, rays_for
from oracle import ops, pipeline


def _scene(name, regime, small=True, act='relu'):
    if name == 'cfgB':
        st = make_state(name, xy=12 if small else 20, depth=10 if small else 16, regime=regime)
        if act != 'relu':
            mpi_act.scale_state_rgbnet(st, act)
    elif name == 'cfg1':
        st = make_state(name, res=10 if small else 16, regime=regime)
        if regime == 'shell':
            # lift the shell into view (as make_cfg1 does for the fog) and raise the threshold: at the coarse stage's
            # 1e-7 the fp32 alpha cannot resolve it (1 + e^x rounds to 1 below x = -17), every sample on the shell's
            # flank would be borderline
            st['density'] = st['density'] + 10.0
            st['fast_color_thres'] = 1e-3
    else:
        st = make_state(name, res=10 if small else 16, regime=regime)
    return st


def _rays(st, H, W, **kw):
    (ro, rd, vd), rkw = rays_for(st, H, W, **kw)
    return ro, rd, vd, rkw


def _oracle(st, ro, rd, vd, kw):
    trace = {}
    out = pipeline.forward(st, ro, rd, vd, ops.CpuOps, trace=trace, **kw)
    return out, trace


@pytest.mark.parametrize('name', ['cfg1', 'cfgA', 'cfgB', 'cfgC'])
@pytest.mark.parametrize('regime', ['fog', 'shell'])
def test_forward_matches_oracle_pipeline(name, regime):
    st = _scene(name, regime, small=False)
    ro, rd, vd, kw = _rays(st, 16, 14, **({'radius': 0.6} if name == 'cfgC' else {}))
    ref, trace = _oracle(st, ro, rd, vd, kw)
    P = R.params_from_state(st)
    ours = R.forward64(P, ro, rd, vd, kw)
    stg = ours['_']
    occ = trace['occupied']
    assert torch.equal(stg['occ_ray_id'], occ['ray_id']) and torch.equal(stg['occ_step_id'], occ['step_id'])
    assert torch.equal(stg['occ_pts'], occ['pts'])
    assert torch.equal(stg['comp_ray_id'], trace['composited']['ray_id'])
    assert torch.equal(ours['ray_id'], ref['ray_id']) and ours['ray_id'].numel() > 0
    # the oracle runs the reference's fp32 arithmetic: it must lie within the fp32 error bounds of train_ref64.Bounds
    # (forward values only: no loss, so the entropy loss's clamp is no threshold here)
    b = R.Bounds(P, ours, torch.zeros(ro.shape[0], 3), ro.shape[0], lw=dict(R.LOSS_WEIGHTS, entropy_last=0.0))
    assert not R.check_margins(P, b, ours), ('borderline sample', R.check_margins(P, b, ours))
    n = ro.shape[0]
    rid = ours['ray_id']
    s = stg['s'].double()
    depth_bound = torch.zeros(n, dtype=torch.float64).index_add_(0, rid, b.weights * s) + \
        (b.n_r + 2) * R.U * torch.zeros(n, dtype=torch.float64).index_add_(0, rid, ours['weights'].detach() * s)
    checks = [('alpha of the occupied samples', stg['alpha_all'], occ['alpha'], b.alpha_occ),
              ('alphainv_last', ours['alphainv_last'], ref['alphainv_last'], b.alphainv_last),
              ('weights', ours['weights'], ref['weights'], b.weights), ('raw_alpha', ours['raw_alpha'], ref['raw_alpha'], b.raw_alpha),
              ('raw_rgb', ours['raw_rgb'], ref['raw_rgb'], b.raw_rgb), ('rgb_marched', ours['rgb_marched'], ref['rgb_marched'], b.rgb_marched),
              ('depth', ours['depth'], ref['depth'], depth_bound)]
    for k, a, r, e in checks:
        a, r = a.detach().double().reshape(-1), r.double().reshape(-1)
        assert a.shape == r.shape, k
        err = (a - r).abs()
        assert (err <= e.reshape(-1)).all(), (k, float((err / e.reshape(-1)).max()))
    if name in ('cfgB', 'cfgC'):
        assert ours['n_max'] == ref['n_max'] and torch.allclose(ours['s'].double(), ref['s'].double(), rtol=0, atol=1e-7)
    if name == 'cfgC':
        assert torch.equal(ours['t'], ref['t']) and torch.equal(ours['step_id'], ref['step_id'])


# ---------------------------------------------------------------------------------------------------------------------
# gradients against central differences
# ---------------------------------------------------------------------------------------------------------------------
FD_CASES = [('cfg1', 'fog', 'relu'), ('cfgA', 'fog', 'relu'), ('cfgA', 'shell', 'relu'), ('cfgB', 'fog', 'relu'),
            ('cfgB', 'fog', 'gauss'), ('cfgB', 'fog', 'lkrelu'), ('cfgC', 'fog', 'relu')]


# rgbper (detached weights) and nearclip (density - density.detach()) define a gradient, not a function of the
# parameters: central differences see only the MSE, entropy and distortion terms
FD_WEIGHTS = dict(R.LOSS_WEIGHTS, rgbper=0.0, nearclip=0.0)


def _loss(P, ro, rd, vd, kw, target):
    out = R.forward64(P, ro, rd, vd, kw, global_step=1, is_train=True)
    return R.composite_loss(out, target, ro.shape[0], near_thres=0.3, weights=FD_WEIGHTS), out


def _fate(out):
    st = out['_']
    return (out['ray_id'].clone(), st['comp_ray_id'].clone(), st['comp_live'].clone())


def _chosen_entries(grid, grad, k=4):
    """Flat indices of up to k entries with non-zero gradient in each of: the 8 corner voxels' neighbourhood (within one
    voxel of a grid corner), the faces (one coordinate at its first / last index) and the interior."""
    C, X, Y, Z = grid.shape[1:]
    ii, jj, kk = torch.meshgrid(torch.arange(X), torch.arange(Y), torch.arange(Z), indexing='ij')
    edge = lambda a, n: (a <= 0) | (a >= n - 1)
    near = lambda a, n: (a <= 1) | (a >= n - 2)
    n_face = edge(ii, X).int() + edge(jj, Y).int() + edge(kk, Z).int()
    corner = near(ii, X) & near(jj, Y) & near(kk, Z)
    cats = [corner, (n_face >= 1) & ~corner, n_face == 0]
    g = grad[0].abs()
    out = []
    for cat in cats:
        sc = torch.where(cat[None].expand(C, -1, -1, -1), g, torch.zeros_like(g)).flatten()
        top = torch.topk(sc, min(k, int((sc > 0).sum())))
        out += top.indices.tolist()
    return out


@pytest.mark.parametrize('name,regime,act', FD_CASES)
def test_gradients_match_central_differences(name, regime, act):
    t0 = time.perf_counter()
    st = _scene(name, regime, small=True, act=act)
    if name == 'cfgC':
        st['k0'] = st['k0'] * 0.5
    ro, rd, vd, kw = _rays(st, 6, 7, **({'radius': 0.6} if name == 'cfgC' else {}))
    kw['rand_bkgd'] = False
    target = torch.rand(ro.shape[0], 3, generator=torch.Generator().manual_seed(0)).double()
    P = R.params_from_state(st, act)
    loss, out = _loss(P, ro, rd, vd, kw, target)
    loss.backward()
    fate = _fate(out)
    params = R.trainable(P)
    checks = []
    for key in ('density.grid', 'k0.grid'):
        p = params[key]
        for i in _chosen_entries(p.detach(), p.grad):
            checks.append((key, i))
    for key in [k for k in params if k.startswith('rgbnet')]:
        p = params[key]
        flat = p.grad.flatten().abs()
        checks += [(key, int(i)) for i in torch.topk(flat, min(2, flat.numel())).indices]
    assert len(checks) >= 12, checks
    worst = 0.0
    for key, i in checks:
        p = params[key]
        an = p.grad.flatten()[i].item()
        h = 1e-6 * max(1.0, abs(p.detach().flatten()[i].item()))
        vals = []
        for sgn in (1, -1):
            with torch.no_grad():
                p.view(-1)[i] += sgn * h
            with torch.enable_grad():
                l, o = _loss(P, ro, rd, vd, kw, target)
            with torch.no_grad():
                p.view(-1)[i] -= sgn * h
            f = _fate(o)
            assert all(torch.equal(a, b) for a, b in zip(f, fate)), ('a difference step changed the sample lists', key, i)
            vals.append(l.item())
        fd = (vals[0] - vals[1]) / (2 * h)
        err = abs(fd - an)
        bound = 1e-6 * max(abs(an), 1e-3 * p.grad.abs().max().item()) + 1e-9
        worst = max(worst, err / bound)
        assert err <= bound, (key, i, an, fd)
    print(f'\n[fd {name} {regime} {act}] {len(checks)} entries, worst err/bound {worst:.3f}, {time.perf_counter() - t0:.2f} s')
