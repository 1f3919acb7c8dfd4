"""GPU: the training forward's gradients (k4nerf/train_forward.py) for all three models against the float64 autograd
restatement of train_ref64.py, element by element, with run_sr.py's composite loss (MSE, entropy on alphainv_last,
nearclip, distortion, rgbper) on both sides.

Each case runs the library, ``m(rays, global_step=1, is_train=True, **kw)``, with forward hooks on ``m.density`` and
``m.k0`` (per-sample points and values, ``retain_grad``), and the restatement on the same fp32 sample points.
Compared: the sample lists (identical ray ids and points; every threshold decision farther from its threshold than the
fp32 error of the compared quantity, else the case fails as "borderline sample"), the per-ray and per-sample forward
values, dL/d(density sample) and dL/d(k0 sample), and the gradients of density.grid, k0.grid and the rgbnet.

Error model (u = 2^-24; every bound is fp64 arithmetic on the restatement's values, train_ref64.Bounds):
  * trilinear lookup: 10u sum_k w_k |g_k| (eight products and the FMA chain) plus the voxel coordinate's rounding,
    5u (size - 1) per axis, times the slope bound 2 max_k |g_k| over the cell's corners.
  * alpha = 1 - (1 + e^x)^-I: |d alpha| <= alpha' E_x + (1 - alpha)(I (3 sigma(x) + 1) u + 8u) + u alpha
    (exp, the add and pow within a few ulp; the pow's relative error is multiplied by I: MPI's I = 256 / depth).
  * transmittance: each factor 1 - alpha_k carries rho_k = |d alpha_k| / (1 - alpha_k) + 2u, so T_i is within
    prod_{k<i} (1 + rho_k) - 1 of the fp64 T_i relatively.  The near-opaque trap is this conditioning term: alpha's
    own rounding u alpha becomes u alpha / (1 - alpha) in 1 - alpha, and it is carried per sample, not spread over all.
  * sums over a ray of n_r samples (rgb_feature, the suffix sum of Alphas2Weights.backward, the distortion loss's
    prefix sums): (n_r + 2) u times the fp64 sum of absolute terms, plus the propagated term errors.
  * the loss's upstream gradients, Alphas2Weights.backward (g_w T - B / (1 - alpha), with B's error and
    B |d alpha| / (1 - alpha)^2) and Raw2Alpha.backward (alpha' relative error u((I+1)(3+|x|)+10) + (1+I) E_x) are
    propagated term by term.
  * rgbnet: per layer (fan_in + 2) u (|W| |h| + |b|) plus |W| E_h forward; backward the same with the transposed
    fan; a ReLU / LeakyReLU unit whose pre-activation is within its error of 0 may take either slope; the Gaussian's
    derivative moves by at most E_z / a^2.  Weight gradients sum over all S shaded samples: (S + 2) u sum |d| |h|.
  * grid gradients: per voxel, the scatter of the per-sample bound with the trilinear weights, plus (2 coordinate
    term + 4u) |g_s| on every corner (the fp32 weights' error), plus (n_v + 2) u sum_s w |g_s| for the order of the
    n_v fp32 atomics that land on the voxel (n_v counted per voxel).
Each case prints its largest observed error as a fraction of its bound.
"""
import time

import pytest
import torch

import mpi_act
import train_ref64 as R
from helpers import make_state, model_from_state
from oracle import pipeline, scenes

pytestmark = pytest.mark.gpu

NEAR_THRES = 0.5            # the DirectContractedVoxGO cases' near_clip / scene_radius


@pytest.fixture
def no_tf32():
    prev = (torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32)
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    yield
    torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32 = prev


# ---------------------------------------------------------------------------------------------------------------------
# cases
# ---------------------------------------------------------------------------------------------------------------------
def _dvgo(xyz_min, xyz_max, res_vox, regime, thres, rgbnet_dim=12, direct=True, pe=4, width=32):
    st = pipeline.dvgo_state(xyz_min, xyz_max, num_voxels=res_vox, num_voxels_base=res_vox, alpha_init=1e-2,
                             fast_color_thres=thres, rgbnet_dim=rgbnet_dim, rgbnet_direct=direct, rgbnet_depth=3,
                             rgbnet_width=width, viewbase_pe=pe)
    scenes.fill_grids(st, regime)
    scenes.fill_rgbnet(st)
    st.update(_num_voxels=res_vox, _num_voxels_base=res_vox, _alpha_init=1e-2)
    return st


def _with_miss_rays(ro, rd, vd, kind, n=7):
    """n more rays that miss the box: pointing away from it (DirectVoxGO) or starting far outside the NDC box."""
    if kind == 'dvgo':
        ro2, rd2 = ro[:n].clone(), -rd[:n]
    else:
        ro2, rd2 = ro[:n].clone(), rd[:n].clone()
        ro2[:, 0] += 50.0
    vd2 = rd2 / rd2.norm(dim=-1, keepdim=True)
    cat = lambda a, b: torch.cat([a, b]).contiguous()
    return cat(ro, ro2), cat(rd, rd2), cat(vd, vd2)


def build_case(cid):
    """(state, act, rays_o, rays_d, viewdirs, render kwargs) of a case; CPU tensors."""
    act = 'relu'
    kw_extra = {}
    if cid.startswith('dvgo'):
        kw = dict(scenes.RENDER_KW_DVGO)
        H, W, cam = 16, 14, {}
        if cid == 'dvgo_direct_fog':
            st = _dvgo([-1, -1, -1], [1, 1, 1], 16 ** 3, 'fog', 1e-4)
        elif cid == 'dvgo_direct_shell':
            st = _dvgo([-1, -1, -1], [1, 1, 1], 16 ** 3, 'shell', 1e-4)
        elif cid == 'dvgo_nondirect_pe0_thres0':
            st = _dvgo([-1, -1, -1], [1, 1, 1], 16 ** 3, 'fog', 0.0, rgbnet_dim=12, direct=False, pe=0)
        elif cid == 'dvgo_nondirect_slab':
            # an opaque slab across the box: rays stop at T < 1e-3 inside it, the fog behind it is past the stop
            st = _dvgo([-1, -1, -1], [1, 1, 1], 16 ** 3, 'fog', 1e-4, rgbnet_dim=12, direct=False, pe=4)
            st['density'][0, 0, 7:9] = 12.0
        elif cid == 'dvgo_cfg1_offcentre':
            # off-centre, non-cubic box and grid (19 x 15 x 7 voxels), no rgbnet
            st = _dvgo([-0.9, -0.5, -0.3], [0.6, 0.7, 0.25], 2200, 'fog', 1e-4, rgbnet_dim=0)
            assert len(set(st['world_size'].tolist())) == 3
        elif cid == 'dvgo_coarse8_1M':
            # an 8^3 grid and ~10^6 samples: every voxel takes thousands of fp32 atomics
            st = _dvgo([-1, -1, -1], [1, 1, 1], 8 ** 3, 'fog', 0.0, rgbnet_dim=0)
            st['density'] = st['density'] * 0.5 - 1.5
            H, W = 336, 336
        else:
            raise ValueError(cid)
        ro, rd, vd = scenes.blender_rays(H, W, **cam)
        ro, rd, vd = _with_miss_rays(ro, rd, vd, 'dvgo')
    elif cid.startswith('mpi'):
        kw = dict(scenes.RENDER_KW_MPI)
        act = cid.split('_')[1]
        if cid.endswith('pe_randbkgd_shell'):
            st = make_state('cfgB', xy=20, depth=16, regime='shell', viewbase_pe=2, spatial_pe=2, width=32)
            kw_extra['rand_bkgd'] = True
        else:
            st = make_state('cfgB', xy=20, depth=16, regime='fog', width=32)
        if act != 'relu':
            mpi_act.scale_state_rgbnet(st, act)
        ro, rd, vd = scenes.llff_rays(16, 13 if kw_extra else 14)
        ro, rd, vd = _with_miss_rays(ro, rd, vd, 'mpi')
    else:
        kw = dict(scenes.RENDER_KW_DCVGO)
        inside = cid == 'dcvgo_inside_fog'
        st = make_state('cfgC', res=16, regime='fog' if inside else 'shell', width=32)
        ro, rd, vd = scenes.blender_rays(16, 14 if inside else 13, radius=0.6 if inside else 4.0)
        extra = scenes.blender_rays(1, 7, radius=0.6 if inside else 4.0)
        ro, rd, vd = (torch.cat([a, b]).contiguous() for a, b in zip((ro, rd, vd), extra))
    kw.update(kw_extra)
    return st, act, ro, rd, vd, kw


CASES = ['dvgo_direct_fog', 'dvgo_direct_shell', 'dvgo_nondirect_pe0_thres0', 'dvgo_nondirect_slab',
         'dvgo_cfg1_offcentre', 'dvgo_coarse8_1M', 'mpi_relu_fog', 'mpi_gauss_fog', 'mpi_lkrelu_fog',
         'mpi_relu_pe_randbkgd_shell', 'dcvgo_inside_fog', 'dcvgo_outside_shell']


def _model(st, act, dev):
    if st['kind'] == 'dmpigo':
        return mpi_act.mpi_model(st, act, dev)
    return model_from_state(st, dev)


# ---------------------------------------------------------------------------------------------------------------------
# the comparison
# ---------------------------------------------------------------------------------------------------------------------
class Ratio:
    def __init__(self):
        self.worst = {}

    def check(self, name, ours, ref, bound):
        a = ours.detach().double().cpu().reshape(-1)
        b = ref.detach().double().cpu().reshape(-1)
        e = bound.detach().double().cpu().reshape(-1)
        assert a.shape == b.shape == e.shape, (name, a.shape, b.shape, e.shape)
        err = (a - b).abs()
        assert torch.isfinite(a).all(), name
        bad = err > e
        if bad.any():
            i = int(torch.nonzero(bad)[0])
            raise AssertionError(f'{name}: {int(bad.sum())} of {a.numel()} elements over their bound; first at {i}: '
                                 f'ours {a[i].item():.9g} ref {b[i].item():.9g} bound {e[i].item():.3g}')
        pos = e > 0
        r = float((err[pos] / e[pos]).max()) if pos.any() else 0.0
        self.worst[name] = max(self.worst.get(name, 0.0), r)


def run_case(cid, dev, seed=0):
    st, act, ro, rd, vd, kw = build_case(cid)
    n = ro.shape[0]
    target = torch.rand(n, 3, generator=torch.Generator().manual_seed(seed))
    m = _model(st, act, dev)
    P = R.params_from_model(m)
    lin = {}
    if m.rgbnet is not None:
        from k4nerf._scene import linear_layers
        names = {id(p): k for k, p in m.named_parameters()}
        for i, l in enumerate(linear_layers(m.rgbnet)):
            lin[names[id(l.weight)]], lin[names[id(l.bias)]] = f'rgbnet.L{i}.weight', f'rgbnet.L{i}.bias'

    # ---- the library
    cap = {}

    def hook(name):
        def f(mod, inp, out):
            out.retain_grad()
            cap[name] = (inp[0].detach().clone(), out)
        return f
    hs = [m.density.register_forward_hook(hook('density')), m.k0.register_forward_hook(hook('k0'))]
    ro_d, rd_d, vd_d = ro.to(dev), rd.to(dev), vd.to(dev)
    torch.cuda.manual_seed(1234)
    out = m(ro_d, rd_d, vd_d, global_step=1, is_train=True, **kw)
    loss = R.composite_loss(out, target.to(dev), n, near_thres=NEAR_THRES)
    loss.backward()
    torch.cuda.synchronize()
    for h in hs:
        h.remove()

    # ---- the restatement
    def rand_bkgd(shape):
        torch.cuda.manual_seed(1234)
        return torch.rand(shape, device=dev, dtype=torch.float32).cpu()
    ref = R.forward64(P, ro, rd, vd, kw, global_step=1, is_train=True, rand_bkgd=rand_bkgd, sample_device=dev)
    loss64 = R.composite_loss(ref, target, n, near_thres=NEAR_THRES)
    loss64.backward()
    b = R.Bounds(P, ref, target, n, near_thres=NEAR_THRES)
    s = ref['_']
    bad = R.check_margins(P, b, ref)
    assert not bad, ('borderline sample: fp32 and fp64 may take it to different fates', cid, bad)

    # ---- sample lists
    q = Ratio()
    assert torch.equal(cap['density'][0].cpu().reshape(-1, 3), s['occ_pts']), 'density sample points'
    assert torch.equal(out['ray_id'].cpu(), ref['ray_id']), 'ray ids of the shaded samples'
    assert torch.equal(cap['k0'][0].cpu().reshape(-1, 3), s['pts']), 'k0 sample points'
    # ---- forward values
    q.check('rgb_marched', out['rgb_marched'], ref['rgb_marched'], b.rgb_marched)
    q.check('alphainv_last', out['alphainv_last'], ref['alphainv_last'], b.alphainv_last)
    q.check('weights', out['weights'], ref['weights'], b.weights)
    q.check('raw_alpha', out['raw_alpha'], ref['raw_alpha'], b.raw_alpha)
    q.check('raw_rgb', out['raw_rgb'], ref['raw_rgb'], b.raw_rgb)
    if st['kind'] != 'dvgo':
        assert out['n_max'] == ref['n_max']
        q.check('s', out['s'], ref['s'], 2 * R.U * ref['s'].double().abs())
    if st['kind'] == 'dcvgo':
        assert torch.equal(out['t'].cpu(), ref['t']) and torch.equal(out['step_id'].cpu(), ref['step_id'])
        inner = s['inner']
        wm = torch.zeros(n, dtype=torch.float64)
        rid = ref['ray_id']
        bw = wm.clone().index_add_(0, rid[inner], b.weights[inner]) + \
            (b.n_r + 2) * R.U * wm.clone().index_add_(0, rid[inner], ref['weights'].detach()[inner])
        q.check('wsum_mid', out['wsum_mid'], ref['wsum_mid'], bw)
    # ---- per-sample gradients
    gd_ours, gd_ref = cap['density'][1].grad.reshape(-1), s['density'].grad
    q.check('dL/d density sample', gd_ours, gd_ref, b.g_density)
    # occupied samples that alpha2weight never reaches (below the alpha threshold, or past the T < 1e-3 stop)
    past = ~torch.zeros_like(s['sel_alpha']).masked_scatter_(s['sel_alpha'], s['comp_live'])
    if st['kind'] != 'dcvgo':          # nearclip adds a constant to DirectContractedVoxGO's raw_density gradient
        assert torch.equal(gd_ours.cpu()[past], torch.zeros_like(gd_ours.cpu()[past])), 'gradient past the stop'
    k0o = cap['k0'][1]
    q.check('dL/d k0 sample', k0o.grad.reshape(k0o.shape[0], -1), s['k0'].grad, b.g_k0)
    # ---- parameter gradients
    ours_g = {lin.get(k, k): p.grad for k, p in m.named_parameters() if p.grad is not None}
    ref_g = {k: p.grad for k, p in R.trainable(P).items() if p.grad is not None}
    assert set(ours_g) == set(ref_g), (sorted(ours_g), sorted(ref_g))
    for k in ref_g:
        q.check(k, ours_g[k], ref_g[k], b.params[k])
    stats = dict(rays=n, samples=int(s['occ_pts'].shape[0]), shaded=int(ref['ray_id'].numel()),
                 past_stop=int((~s['comp_live']).sum()), one_sample_rays=int((torch.bincount(ref['ray_id'], minlength=n) == 1).sum()),
                 empty_rays=int((torch.bincount(s['occ_ray_id'], minlength=n) == 0).sum()),
                 max_atomics=int(b.count_density.max()) if b.count_density.numel() else 0)
    return q.worst, stats


@pytest.mark.parametrize('cid', CASES)
def test_gradients_match_float64_restatement(cuda_device, no_tf32, cid):
    t0 = time.perf_counter()
    worst, stats = run_case(cid, cuda_device)
    top = max(worst.values())
    print(f'\n[train_grad {cid}] worst observed/bound {top:.3g} ({max(worst, key=worst.get)}); {stats}; '
          f'{time.perf_counter() - t0:.1f} s')
    if not cid.startswith('dcvgo'):                 # the appended rays miss the box (the contracted space has no outside)
        assert stats['empty_rays'] >= 7
    if cid != 'dcvgo_inside_fog':                   # rays that graze the scene with exactly one shaded sample
        assert stats['one_sample_rays'] > 0
    if cid == 'dvgo_nondirect_slab':
        assert stats['past_stop'] > 0
    if cid == 'dvgo_coarse8_1M':
        assert stats['samples'] >= 800_000 and stats['max_atomics'] >= 1000


def test_all_miss_batch(cuda_device, no_tf32):
    """Every ray misses the box: forward and backward complete, every gradient is zero, and the library and the
    restatement agree on which parameters receive one."""
    st, act, ro, rd, vd, kw = build_case('dvgo_direct_fog')
    ro, rd = ro[:40].clone(), -rd[:40]
    vd = rd / rd.norm(dim=-1, keepdim=True)
    m = _model(st, act, cuda_device)
    P = R.params_from_model(m)
    target = torch.rand(40, 3, generator=torch.Generator().manual_seed(0))
    out = m(ro.to(cuda_device), rd.to(cuda_device), vd.to(cuda_device), global_step=1, is_train=True, **kw)
    assert out['ray_id'].numel() == 0
    R.composite_loss(out, target.to(cuda_device), 40).backward()
    torch.cuda.synchronize()
    ref = R.forward64(P, ro, rd, vd, kw, global_step=1, is_train=True)
    R.composite_loss(ref, target, 40).backward()
    assert torch.equal(out['alphainv_last'].cpu(), torch.ones(40))
    from k4nerf._scene import linear_layers
    names = {id(p): k for k, p in m.named_parameters()}
    lin = {}
    for i, l in enumerate(linear_layers(m.rgbnet)):
        lin[names[id(l.weight)]], lin[names[id(l.bias)]] = f'rgbnet.L{i}.weight', f'rgbnet.L{i}.bias'
    ours = {lin.get(k, k): p.grad for k, p in m.named_parameters() if p.grad is not None}
    theirs = {k: p.grad for k, p in R.trainable(P).items() if p.grad is not None}
    assert set(ours) == set(theirs), (sorted(ours), sorted(theirs))
    for k, g in ours.items():
        assert torch.count_nonzero(g) == 0 and torch.count_nonzero(theirs[k]) == 0, k


# ---------------------------------------------------------------------------------------------------------------------
# the bars see real mistakes: Python-level changes of the library's backward must make a case fail
# ---------------------------------------------------------------------------------------------------------------------
def _patch_alphas2weights_drop_last(monkeypatch):
    from k4nerf import autograd_ops
    orig = autograd_ops.Alphas2Weights.backward

    def backward(ctx, grad_weights, grad_last):
        return orig(ctx, grad_weights, torch.zeros_like(grad_last))
    monkeypatch.setattr(autograd_ops.Alphas2Weights, 'backward', staticmethod(backward))


def _patch_grid_backward(monkeypatch, fn):
    from k4nerf import grid
    orig = grid._GridSample.backward

    def backward(ctx, grad_out):
        g, *rest = orig(ctx, grad_out)
        return (fn(g), *rest)
    monkeypatch.setattr(grid._GridSample, 'backward', staticmethod(backward))


def _patch_raw2alpha_interval_one(monkeypatch):
    from k4nerf import autograd_ops, render_utils_cuda

    def backward(ctx, grad_alpha):
        (e,) = ctx.saved_tensors
        return render_utils_cuda.raw2alpha_backward(e, grad_alpha.contiguous(), 1.0), None, None
    monkeypatch.setattr(autograd_ops.Raw2Alpha, 'backward', staticmethod(backward))


def _swap01(g):
    if g.shape[1] < 2:
        return g
    g = g.clone()
    g[:, [0, 1]] = g[:, [1, 0]]
    return g


SENSITIVITY = {
    'alphas2weights_drops_grad_last': ('dvgo_direct_fog', _patch_alphas2weights_drop_last),
    'grid_scatter_mirrored_x': ('dvgo_cfg1_offcentre', lambda mp: _patch_grid_backward(mp, lambda g: g.flip(2))),
    'k0_scatter_channels_swapped': ('dvgo_direct_fog', lambda mp: _patch_grid_backward(mp, _swap01)),
    'raw2alpha_interval_one': ('mpi_relu_fog', _patch_raw2alpha_interval_one),
}


@pytest.mark.parametrize('which', sorted(SENSITIVITY))
def test_comparison_fails_on_a_wrong_backward(cuda_device, no_tf32, monkeypatch, which):
    cid, patch = SENSITIVITY[which]
    patch(monkeypatch)
    with pytest.raises(AssertionError) as e:
        run_case(cid, cuda_device)
    print(f'\n[train_grad sensitivity {which}] {str(e.value).splitlines()[0][:160]}')


# ---------------------------------------------------------------------------------------------------------------------
# cumdist_thres (csrc/k4_train.cu) against the oracle, bit-exact
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('shape', [(1, 1), (3, 1), (7, 40), (5000, 37)])
@pytest.mark.parametrize('thres', [0.0, 0.05, 1e30])
def test_cumdist_thres_matches_oracle(cuda_device, shape, thres):
    from k4nerf import render_utils_cuda
    from oracle.ops import CpuOps
    g = torch.Generator().manual_seed(shape[0] * 131 + shape[1])
    dist = torch.rand(shape, generator=g) * 0.03
    dist[torch.rand(shape, generator=g) < 0.2] = 0.0            # repeated points (zero distances)
    ours = render_utils_cuda.cumdist_thres(dist.to(cuda_device).contiguous(), thres).cpu()
    ref = CpuOps.cumdist_thres(dist, thres)
    assert ours.dtype == torch.bool and ours.shape == ref.shape
    assert torch.equal(ours, ref)
    if thres == 0.0:
        assert torch.equal(ref, dist > 0)
    if thres == 1e30:
        assert not ref.any()
