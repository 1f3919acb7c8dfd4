"""GPU: the fused training step (k4nerf.train_fused.render_loss, csrc/k4_train_march.cu) at the shapes the reference's
configs train with, at the largest rgbnet it accepts, at warp and loss-reduction structures the scenes of
test_gpu_train_fused.py only reach by accident, and with frozen parameters.  Every case is held to the float64
restatement within test_gpu_train_fused.compare's bounds (that file's docstring has the error model): rgb_marched,
alphainv_last, each loss term, the total and the gradients of density.grid, k0.grid and the six rgbnet tensors.

The backward's rgbnet weight gradients are summed per warp from rows staged in shared memory with strides
ks = max(dim0, width) + 1 (layer inputs) and ds = width + 1 (output deltas), so the limit cases assert the dim0, width,
ks and ds they are built for, and the warp cases assert their hit pattern from the restatement's ray ids.
Each case prints its largest observed error as a fraction of its bound.
"""
import pytest
import torch

import mpi_act
import train_ref64 as R
from test_gpu_train_fused import _grads, compare, fused_extra, reference, run_fused, term_refs
from test_gpu_train_grad import Ratio, _model, no_tf32  # noqa: F401  (fixture)
from helpers import make_state
from oracle import scenes

pytestmark = pytest.mark.gpu

FULL = dict(main=1.0, entropy_last=0.01, distortion=0.01, rgbper=0.1)
SYN_FINE_LW = dict(main=1.0, entropy_last=0.001, distortion=0.0, rgbper=0.01)         # configs/default.py fine_train
FERN_LW = dict(main=1.0, entropy_last=0.001, distortion=0.01, rgbper=0.1)             # llff_default_lg + fern_lg_joint_l1
TM_T = 32                       # rays per CTA of the fused kernels: one warp
TM_RED_T = 1024                 # threads of the one-CTA loss reduction


# ---------------------------------------------------------------------------------------------------------------------
# rays
# ---------------------------------------------------------------------------------------------------------------------
def _miss(ro, rd, vd, kind, idx):
    """The rays at idx miss the box: reversed (DirectVoxGO, the camera is outside it) or moved far off the NDC box."""
    ro, rd, vd = ro.clone(), rd.clone(), vd.clone()
    if kind == 'dvgo':
        rd[idx] = -rd[idx]
        vd[idx] = -vd[idx]
    else:
        ro[idx, 0] += 50.0
    return ro.contiguous(), rd.contiguous(), vd.contiguous()


def _spread_misses(ro, rd, vd, kind, frac=16, seed=0):
    n = ro.shape[0]
    idx = torch.randperm(n, generator=torch.Generator().manual_seed(seed))[:n // frac]
    return _miss(ro, rd, vd, kind, idx)


def _dvgo_rays(n, seed=0):
    """n rays from 4-5 units outside the [-1, 1]^3 box, each through a point inside [-0.8, 0.8]^3: every ray hits."""
    g = torch.Generator().manual_seed(seed)
    tgt = torch.rand(n, 3, generator=g) * 1.6 - 0.8
    ro = torch.tensor([0.4, -4.0, 1.2]) + torch.rand(n, 3, generator=g) * 0.6
    rd = tgt - ro
    rd = rd / rd.norm(dim=-1, keepdim=True)
    return ro.contiguous(), rd.contiguous(), rd.clone()


def _mpi_rays(n, seed=0):
    """n NDC rays from z = -1 to z = 1 that stay inside the box's x / y extent: every ray takes every step."""
    g = torch.Generator().manual_seed(seed)
    ro = torch.cat([torch.rand(n, 2, generator=g) * 2 - 1, -torch.ones(n, 1)], 1)
    rd = torch.cat([torch.rand(n, 2, generator=g) * 0.6 - 0.3, torch.full((n, 1), 2.0)], 1)
    vd = torch.cat([rd[:, :2], -torch.ones(n, 1)], 1)
    return ro.contiguous(), rd.contiguous(), (vd / vd.norm(dim=-1, keepdim=True)).contiguous()


def _graze_rays(kind):
    """One warp: lane 0 crosses the whole grid, lanes 1..31 clip a corner (DirectVoxGO: the x = y = 1 edge; DirectMPIGO:
    they start just inside x = 1.5 and leave through it within one or two planes)."""
    k = torch.arange(31, dtype=torch.float32)
    if kind == 'dvgo':
        d0 = torch.tensor([1.0, 1.0, 1.0]) / 3 ** 0.5
        ro0 = torch.tensor([0.01, 0.02, -0.015]) - 5.0 * d0
        d = torch.tensor([1.0, -1.0, 0.0]) / 2 ** 0.5
        delta = 0.05 + 0.002 * k                          # the ray's line x + y = 2 - delta: a chord of sqrt(2) delta
        p = torch.stack([1 - delta / 2, 1 - delta / 2, -0.9 + 0.06 * k], 1)
        ro = torch.cat([ro0[None], p - 5.0 * d]).contiguous()
        rd = torch.cat([d0[None], d.expand(31, 3)]).contiguous()
        return ro, rd, rd.clone()
    ro0, rd0 = torch.tensor([0.1, 0.05, -1.0]), torch.tensor([0.2, 0.1, 2.0])
    ro = torch.stack([1.38 + 0.002 * k, -1.5 + 0.1 * k, -torch.ones(31)], 1)
    rd = torch.tensor([3.0, 0.0, 2.0]).expand(31, 3)
    ro, rd = torch.cat([ro0[None], ro]).contiguous(), torch.cat([rd0[None], rd]).contiguous()
    vd = torch.cat([rd[:, :2], -torch.ones(32, 1)], 1)
    return ro, rd, (vd / vd.norm(dim=-1, keepdim=True)).contiguous()


# ---------------------------------------------------------------------------------------------------------------------
# scenes
# ---------------------------------------------------------------------------------------------------------------------
def _mpi(act='relu', calm=False, **kw):
    """calm: fast_color_thres 0 and the fog shifted down by 2, as test_larger_mpi_case: at 32 planes and a few hundred
    rays some sample otherwise sits too close to the weight threshold or the T < 1e-3 stop for the margin check."""
    st = make_state('cfgB', **dict(dict(xy=20, depth=16, regime='fog'), **kw))
    if calm:
        st['fast_color_thres'] = 0.0
        st['density'] = st['density'] - 2.0
    if act != 'relu':
        mpi_act.scale_state_rgbnet(st, act)
    return st


def _dvgo(**kw):
    return make_state('cfgA', **dict(dict(res=20, regime='fog'), **kw))


def _kw(st, rand_bkgd=False):
    kw = dict(scenes.RENDER_KW_DVGO if st['kind'] == 'dvgo' else scenes.RENDER_KW_MPI)
    if rand_bkgd:
        kw['rand_bkgd'] = True
    return kw


def _lw(st, lw):
    return dict(lw, distortion=0.0) if st['kind'] == 'dvgo' else dict(lw)


def rgbnet_shape(m):
    """(dim0, width, ks, ds) of the model's rgbnet: dim0 checked against the model's input formula, ks / ds as tm_params
    computes them."""
    from k4nerf import _lib
    from k4nerf._scene import linear_layers
    layers = linear_layers(m.rgbnet)
    dim0, width = layers[0].in_features, layers[0].out_features
    mpi = m._k4_kind == _lib.K4_KIND_DMPIGO
    off = 3 if (not mpi and not m.rgbnet_direct) else 0
    assert dim0 == int(m.k0.grid.shape[1]) - off + 3 + 6 * m.viewbase_pe + (3 + 6 * m.spatial_pe if mpi else 0)
    return dim0, width, max(dim0, width) + 1, width + 1


def run(st, act, ro, rd, vd, kw, lw, dev, seed=0, freeze=()):
    """The fused step and the restatement on one scene; returns (worst ratios, restatement, bounds, fused outputs,
    model).
    freeze: 'k0' and / or 'rgbnet0' (the first Linear's weight and bias) are set requires_grad_(False) on the model."""
    from k4nerf._scene import linear_layers
    target = torch.rand(ro.shape[0], 3, generator=torch.Generator().manual_seed(seed))
    m = _model(st, act, dev)
    frozen = {'k0': [(m.k0.grid, 'k0.grid')]}
    if m.rgbnet is not None:
        l0 = linear_layers(m.rgbnet)[0]
        frozen['rgbnet0'] = [(l0.weight, 'rgbnet.L0.weight'), (l0.bias, 'rgbnet.L0.bias')]
    off = [pn for f in freeze for pn in frozen[f]]
    for p, _ in off:
        p.requires_grad_(False)
    P = R.params_from_model(m)
    loss, out = run_fused(m, ro, rd, vd, target, kw, lw, dev)
    ref, b = reference(P, ro, rd, vd, target, kw, lw, dev)
    tr = R.trainable(P)
    for p, name in off:
        assert p.grad is None, name
        tr[name].grad = None                    # the restatement differentiates everything; drop what the model froze
    q = Ratio()
    compare(m, P, ref, b, out, loss, target, lw, q, extra=fused_extra(P, ref, b, target, lw))
    return q.worst, ref, b, out, m


def _report(tag, worst, extra=''):
    top = max(worst.values())
    mlp = {k: v for k, v in worst.items() if k.startswith('rgbnet')}
    if mlp:
        extra = f'; rgbnet worst {max(mlp.values()):.3g} ({max(mlp, key=mlp.get)})' + extra
    print(f'\n[train_fused_shapes {tag}] worst observed/bound {top:.3g} ({max(worst, key=worst.get)}){extra}')
    assert top <= 1.0


# ---------------------------------------------------------------------------------------------------------------------
# 1. the configurations the reference trains with
# ---------------------------------------------------------------------------------------------------------------------
def config_case(cid):
    """(state, act, rays, render kwargs, loss weights) of a reference training configuration.  The fog's density is
    N(0, 0.25^2): alpha then stays within a factor e of alpha_init (DirectVoxGO) or of the MPI bias grid's uniform
    weights (DirectMPIGO), so every alpha and weight is 2x or more from fast_color_thres and no ray reaches T < 1e-3.
    At these sample counts the wider fog of the small scenes puts some sample within its fp32 error of a threshold."""
    if cid.startswith('syn'):
        pe = 0 if cid == 'syn_1x' else 4
        st = make_state('cfgA', res=160, regime='fog', width=128, k0_dim=12, viewbase_pe=pe,
                        rgbnet_direct=cid != 'syn_diffuse')
        st['density'] = st['density'] * 0.25
        ro, rd, vd = _spread_misses(*scenes.blender_rays(32, 48), 'dvgo')
        return st, 'relu', (ro, rd, vd), _kw(st), SYN_FINE_LW
    assert cid == 'llff_fern'
    st = make_state('cfgB', xy=96, depth=256, regime='fog', width=64, k0_dim=9, viewbase_pe=0, spatial_pe=0)
    st['density'] = st['density'] * 0.125                 # fill_grids' MPI fog is 2 N(0, 1)
    ro, rd, vd = _spread_misses(*scenes.llff_rays(32, 48), 'mpi')
    return st, 'relu', (ro, rd, vd), _kw(st, rand_bkgd=True), FERN_LW


CONFIG_SHAPES = {'syn_fine': (39, 128), 'syn_1x': (15, 128), 'syn_diffuse': (36, 128), 'llff_fern': (15, 64)}


@pytest.mark.parametrize('cid', sorted(CONFIG_SHAPES))
def test_reference_configurations(cuda_device, no_tf32, cid):
    st, act, rays, kw, lw = config_case(cid)
    worst, ref, b, out, m = run(st, act, *rays, kw, lw, cuda_device)
    assert rgbnet_shape(m)[:2] == CONFIG_SHAPES[cid]
    if cid.startswith('syn'):
        assert tuple(st['world_size'].tolist()) == (160, 160, 160) and float(m.fast_color_thres) == 1e-4
    else:
        assert int(m.mpi_depth) == 256 and ref['n_max'] == 256
    n_miss = int((torch.bincount(ref['ray_id'], minlength=rays[0].shape[0]) == 0).sum())
    assert n_miss >= rays[0].shape[0] // 16
    _report(cid, worst, f'; {ref["ray_id"].numel()} shaded samples, {n_miss} rays without one')


# ---------------------------------------------------------------------------------------------------------------------
# 2. the kernel's limits and the shapes between them: (scene, act, (dim0, width, ks, ds))
# ---------------------------------------------------------------------------------------------------------------------
LIMITS = {
    # MLP input 32 + 33 + 63 = 128 = K4_MAX_DIM0 at width 128: both strides 129, the largest shared memory
    'mpi_dim0_128_w128': (lambda: _mpi(k0_dim=32, spatial_pe=5, viewbase_pe=10, width=128), 'relu', (128, 128, 129, 129)),
    'dvgo_k0_32_pe10_w128': (lambda: _dvgo(k0_dim=32, viewbase_pe=10, width=128), 'relu', (95, 128, 129, 129)),
    # ks from the input, not the width
    'mpi_dim0_128_w40': (lambda: _mpi(k0_dim=32, spatial_pe=5, viewbase_pe=10, width=40), 'relu', (128, 40, 129, 41)),
    'dvgo_w96': (lambda: _dvgo(k0_dim=12, viewbase_pe=4, width=96), 'relu', (39, 96, 97, 97)),
    'dvgo_diffuse_w127': (lambda: _dvgo(k0_dim=12, viewbase_pe=4, width=127, rgbnet_direct=False), 'relu',
                          (36, 127, 128, 128)),
    'mpi_w127': (lambda: _mpi(k0_dim=9, spatial_pe=2, viewbase_pe=2, width=127), 'relu', (39, 127, 128, 128)),
    'mpi_gauss_w128': (lambda: _mpi('gauss', k0_dim=12, spatial_pe=2, viewbase_pe=2, width=128), 'gauss',
                       (42, 128, 129, 129)),
    'mpi_lkrelu_w128': (lambda: _mpi('lkrelu', k0_dim=12, spatial_pe=2, viewbase_pe=2, width=128), 'lkrelu',
                        (42, 128, 129, 129)),
}


def limit_rays(st):
    if st['kind'] == 'dvgo':
        return _spread_misses(*scenes.blender_rays(16, 16), 'dvgo')
    return _spread_misses(*scenes.llff_rays(16, 14), 'mpi')


@pytest.mark.parametrize('cid', sorted(LIMITS))
def test_rgbnet_limits(cuda_device, no_tf32, cid):
    make, act, shape = LIMITS[cid]
    st = make()
    worst, ref, b, out, m = run(st, act, *limit_rays(st), _kw(st), _lw(st, FULL), cuda_device)
    assert rgbnet_shape(m) == shape
    assert ref['ray_id'].numel() > 1000
    _report(cid, worst, f'; dim0, width, ks, ds = {shape}')


# ---------------------------------------------------------------------------------------------------------------------
# 3. warp and loss-reduction structure
# ---------------------------------------------------------------------------------------------------------------------
def warp_scene(kind):
    if kind == 'dvgo':
        return _dvgo(k0_dim=12, viewbase_pe=4, width=64)
    return _mpi(calm=True, depth=32, k0_dim=9, spatial_pe=2, viewbase_pe=2, width=64)


def warp_case(kind, which):
    """(rays, the set of ray indices that must shade)."""
    base = _dvgo_rays if kind == 'dvgo' else _mpi_rays
    if which.startswith('n'):
        n = int(which[1:])
        return base(n), set(range(n))
    if which == 'lane5':
        n = 8 * TM_T
        miss = torch.tensor([r for r in range(n) if r % TM_T != 5])
        return _miss(*base(n), kind, miss), set(range(5, n, TM_T))
    if which == 'alternate':
        n = 4 * TM_T + 7
        return _miss(*base(n), kind, torch.arange(1, n, 2)), set(range(0, n, 2))
    assert which == 'graze'
    return _graze_rays(kind), set(range(TM_T))


@pytest.mark.parametrize('which', ['n1', 'n31', 'n33', 'lane5', 'alternate', 'graze'])
@pytest.mark.parametrize('kind', ['dmpigo', 'dvgo'])
def test_warp_structure(cuda_device, no_tf32, kind, which):
    st = warp_scene(kind)
    rays, hits = warp_case(kind, which)
    worst, ref, b, out, m = run(st, 'relu', *rays, _kw(st), _lw(st, FULL), cuda_device)
    assert rgbnet_shape(m)[1] == 64
    assert set(ref['ray_id'].unique().tolist()) == hits
    extra = ''
    if which == 'graze':
        steps = torch.bincount(ref['_']['occ_ray_id'], minlength=TM_T)
        assert int(steps[1:].min()) >= 1 and int(steps[0]) >= 10 * int(steps[1:].max()), steps.tolist()
        extra = f'; steps {int(steps[0])} against at most {int(steps[1:].max())}'
    _report(f'{kind} {which}', worst, extra)


def test_distortion_divisor_from_a_late_thread(cuda_device, no_tf32):
    """3000 rays, every one after ray 1700 misses: flatten_eff_distloss divides by ray_id.max() + 1 = 1701.  The loss
    CTA's threads take ceil(3000 / 1024) = 3 rays each, so that maximum is found by thread 566, not by thread 0."""
    n, last = 3000, 1700
    st = warp_scene('dmpigo')
    ro, rd, vd = _miss(*_mpi_rays(n), 'mpi', torch.arange(last + 1, n))
    lw = dict(FULL)
    worst, ref, b, out, m = run(st, 'relu', ro, rd, vd, _kw(st), lw, cuda_device)
    assert int(ref['ray_id'].max()) == last and set(ref['ray_id'].unique().tolist()) == set(range(last + 1))
    chunk = -(-n // TM_RED_T)
    assert last // chunk == 566
    # the check above holds loss_distortion to its bound; it would not hold with another divisor
    target = torch.rand(n, 3, generator=torch.Generator().manual_seed(0))
    v, bd = term_refs(R.params_from_model(m), ref, b, target, lw)['loss_distortion']
    v, bd = float(v), float(bd)
    got = float(out['loss_distortion'])
    for wrong in (n, chunk):                    # all rays, or thread 0's own maximum (ray chunk - 1)
        assert abs(v * (last + 1) / wrong - v) > 2 * bd
    assert abs(got - v) <= bd
    _report('distortion divisor 1701', worst, f'; loss_distortion {got:.9g} (restatement {v:.9g})')


# ---------------------------------------------------------------------------------------------------------------------
# 4. partly frozen parameters: null gradient pointers
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('freeze', ['k0', 'rgbnet0'])
def test_frozen_parameters(cuda_device, no_tf32, freeze):
    st = _mpi(k0_dim=12, spatial_pe=2, viewbase_pe=2, width=128)
    worst, ref, b, out, m = run(st, 'relu', *limit_rays(st), _kw(st), FULL, cuda_device, freeze=(freeze,))
    g = _grads(m)
    expect = {'density.grid', 'k0.grid'} | {f'rgbnet.L{i}.{w}' for i in range(3) for w in ('weight', 'bias')}
    expect -= {'k0.grid'} if freeze == 'k0' else {'rgbnet.L0.weight', 'rgbnet.L0.bias'}
    assert set(g) == expect
    assert all(torch.count_nonzero(v) > 0 for v in g.values())
    _report(f'frozen {freeze}', worst)
