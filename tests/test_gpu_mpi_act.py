"""GPU: DirectMPIGO with act_type 'gauss' / 'lkrelu' in every marcher mode.

1. Per sample (k4_testing_rgbnet): every mode each MPI shape has, on ws configs 6, 7, 8 and on a model padded into
   config 6 (width 48, 7 k0 channels: its padded hidden units have gauss(0) = 1 and must meet zero outgoing weights),
   against the fp64 model within the error model of mpi_act.act_logit_bound.
2. Per ray: every mode against fp32 mode (as test_gpu_march_mlp.check_per_ray_against_fp32), ws also on scenes of its
   own in both ray orders, and the geometry (S_m, S_d, alphainv_last) bit-identical to the relu model of the same grids.
3. At scale: the [384,384,256] LLFF model at 1008x756 against the reference's kernels + ATen (oracle on RefExtOps).
4. End to end: a gauss checkpoint through utils.load_model and render_viewpoints with NDC rays; forward under autograd.
Every scene's rgbnet is scaled so that the activation is exercised (mpi_act.scale_for_act / assert_exercised).
"""
import ctypes as C
import math
import os
import types

import numpy as np
import pytest
import torch

import mpi_act
from helpers import make_state, model_from_state, ref_forward_chunked, rays_for
from march_bounds import FEAT_REL, SIG_REL, U, dim0_of, shape_info, sig, supports
from mpi_act import ACTS, act_logit_bound, assert_exercised, mpi_model, oracle_act, scale_state_rgbnet

pytestmark = pytest.mark.gpu

MODES = {'fp32': 0, 'f16': 1, 'f16x3': 2, 'ws': 4}
ROWS = [1, 33, 64, 128, 300]
# (name, kind, C, vpe, spe, width, direct, config id)
SHAPES = [('cfg6', 'cfgB', 9, 0, 0, 64, 1, 6), ('cfg7', 'cfgB', 12, 4, 0, 128, 1, 7), ('cfg8', 'cfgB', 12, 4, 5, 128, 1, 8),
          ('C7-w48-on6', 'cfgB', 7, 0, 0, 48, 1, 6)]


class ActModel:
    """A small MPI scene with the given rgbnet (fp64 numpy (W, b) pairs, fp32 values) and activation."""

    def __init__(self, spec, layers, act, dev):
        name, kind, c, vpe, spe, w, direct, cid = spec
        st = make_state('cfgB', xy=8, depth=8, regime='fog', k0_dim=c, viewbase_pe=vpe, spatial_pe=spe, width=w)
        st['rgbnet'] = [(torch.tensor(W, dtype=torch.float32), torch.tensor(b, dtype=torch.float32)) for W, b in layers]
        self.layers = [(W.double().numpy(), b.double().numpy()) for W, b in st['rgbnet']]
        self.m = mpi_model(st, act, dev)
        self.spec, self.dev, self.width, self.act = spec, dev, w, act
        shape_info(self, spec)

    def run(self, mode, x, w, owner):
        from k4nerf import _lib
        n = x.shape[0]
        t = lambda a, dt: torch.tensor(np.ascontiguousarray(a), dtype=dt, device=self.dev)
        tx, tw, to = t(x, torch.float32), t(w, torch.float32), t(owner, torch.int32)
        racc = torch.full(((n + 31) // 32 * 32 * 3 + 128 * 3,), float('nan'), device=self.dev)
        a = _lib.RgbnetTestArgs()
        a.mode, a.n = MODES[mode], n
        a.d_x, a.d_w, a.d_owner, a.d_racc, a.d_diffuse = tx.data_ptr(), tw.data_ptr(), to.data_ptr(), racc.data_ptr(), None
        g = C.c_int32(0)
        st = _lib.lib.k4_testing_rgbnet(self.m._get_scene().ptr, C.byref(a), C.byref(g),
                                         C.c_void_p(torch.cuda.current_stream().cuda_stream))
        assert st == 0, (self.spec[0], mode, st, _lib.lib.k4_last_cuda_error().decode())
        G = g.value
        ng = (n + G - 1) // G
        return racc[:ng * G * 3].view(ng, G, 3).double().cpu().numpy(), G


def _inputs(kind, c, vpe, spe, n, rng):
    def emb(v, nf):
        f = 2.0 ** np.arange(nf)
        return np.concatenate([v, np.sin(v[:, :, None] * f).reshape(n, -1), np.cos(v[:, :, None] * f).reshape(n, -1)], 1)
    d = rng.standard_normal((n, 3))
    d /= np.linalg.norm(d, axis=1, keepdims=True)
    x = np.concatenate([rng.standard_normal((n, c)), emb(rng.uniform(-1, 1, (n, 3)), spe), emb(d, vpe)], 1)
    return x.astype(np.float32).astype(np.float64)


def _random_layers(dim0, width, seed):
    torch.manual_seed(seed)
    ls = [torch.nn.Linear(dim0, width), torch.nn.Linear(width, width), torch.nn.Linear(width, 3)]
    return [(l.weight.detach().double().numpy(), l.bias.detach().double().numpy()) for l in ls]


def _racc_check(mode, m, x, w, owner, G, racc):
    """As test_gpu_march_mlp.racc_check, with the activation's error model; returns the largest error / bound."""
    lg, E = act_logit_bound(mode, m, x, None, m.act)
    zc = np.clip(0.0, lg - E, lg + E)
    dmax = sig(zc) * (1 - sig(zc))
    s_hi = sig(lg + E)
    ng = racc.shape[0]
    g = np.arange(x.shape[0]) // G
    ref, bnd, hi, cnt = (np.zeros((ng, G, 3)) for _ in range(4))
    np.add.at(ref, (g, owner), w[:, None] * sig(lg))
    np.add.at(bnd, (g, owner), w[:, None] * (dmax * E + 3.5 * 2.0 ** -23 * s_hi))
    np.add.at(hi, (g, owner), w[:, None] * s_hi)
    np.add.at(cnt, (g, owner), 1.0)
    bnd += np.maximum(cnt - 1, 0) * U * hi
    err = np.abs(racc - ref)
    ok = (err <= bnd) & np.isfinite(racc)
    assert ok.all(), (mode, int((~ok).sum()), float((err / np.maximum(bnd, 1e-300)).max()))
    return float((err / np.maximum(bnd, 1e-300)).max())


# ---------------------------------------------------------------------------------------------------------------------
# 1. per sample
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('act', ACTS)
@pytest.mark.parametrize('spec', SHAPES, ids=[s[0] for s in SHAPES])
def test_every_mode_per_sample_within_bound(cuda_device, spec, act):
    rng = np.random.default_rng(7)
    name, kind, c, vpe, spe, width, direct, cid = spec
    dim0 = dim0_of(kind, c, vpe, spe, direct)
    x = _inputs(kind, c, vpe, spe, 300, rng)
    layers = mpi_act.scale_for_act(_random_layers(dim0, width, seed=cid + 100 * width + dim0), x, act)
    assert_exercised(layers, x, act)
    m = ActModel(spec, layers, act, cuda_device)
    assert _lib_ws_config(m) == cid
    w = np.maximum(rng.random(300), 1e-3).astype(np.float32).astype(np.float64)
    ratios = {}
    for mode in MODES:
        if not supports(spec, mode):
            continue
        for n in ROWS:
            xs, ws = x[:n], w[:n]
            G = 128 if mode == 'ws' else 32
            for owner in (np.concatenate([rng.permutation(G)[:min(G, n - s)] for s in range(0, n, G)]).astype(np.int32),
                          rng.integers(0, 3, size=n).astype(np.int32)):
                racc, Gk = m.run(mode, xs, ws, owner)
                assert Gk == G
                ratios[mode] = max(ratios.get(mode, 0.0), _racc_check(mode, m, xs, ws, owner, G, racc))
    assert {'fp32', 'ws'} <= set(ratios)
    print(name, act, 'largest error/bound', {k: f'{v:.3g}' for k, v in ratios.items()})


def _lib_ws_config(m):
    from k4nerf import _lib
    return _lib.lib.k4_scene_ws_config(m.m._get_scene().ptr)


# ---------------------------------------------------------------------------------------------------------------------
# 2. per ray
# ---------------------------------------------------------------------------------------------------------------------
RAY_SHAPES = [(dict(k0_dim=9, viewbase_pe=0, spatial_pe=0, width=64), 6), (dict(k0_dim=12, viewbase_pe=4, spatial_pe=5, width=128), 8)]


@pytest.mark.parametrize('act', ACTS)
@pytest.mark.parametrize('skw,cfg_id', RAY_SHAPES, ids=['llff', 'cfg8'])
def test_every_mode_against_fp32_per_ray(cuda_device, skw, cfg_id, act):
    """The bound of test_gpu_march_mlp.check_per_ray_against_fp32 with the activation's error model, and the
    geometry of every mode bit-identical to the relu model of the same grids."""
    from oracle import ops, pipeline
    dev = cuda_device
    st = make_state('cfgB', xy=40, depth=24, regime='fog', **skw)
    scale_state_rgbnet(st, act)
    hw = (24, 32)
    (ro, rd, vd), kw = rays_for(st, *hw)
    stats, trace = {}, {}
    with oracle_act(act):
        pipeline.forward(st, ro, rd, vd, ops.CpuOps, stats=stats, trace=trace, **kw)
    m = mpi_model(st, act, dev)
    relu = model_from_state(st, dev)
    spec = ('ray', 'cfgB', skw['k0_dim'], skw['viewbase_pe'], skw['spatial_pe'], skw['width'], 1, cfg_id)
    outs, routs = {}, {}
    args = (ro.to(dev), rd.to(dev), vd.to(dev), kw)
    for mode in MODES:
        if supports(spec, mode):
            outs[mode] = m.render_rays(*args, image_hw=hw, mlp_mode=mode, debug=True)
            routs[mode] = relu.render_rays(*args, image_hw=hw, mlp_mode=mode, debug=True)
    torch.cuda.synchronize()
    outs = {k: {n: t.cpu() for n, t in o.items()} for k, o in outs.items()}
    for mode, o in outs.items():
        r = routs[mode]
        assert torch.equal(o['alphainv_last'], r['alphainv_last'].cpu()), mode
        assert torch.equal(o['ray_stats'], r['ray_stats'].cpu()), mode
        assert torch.equal(o['depth'], r['depth'].cpu()), mode
    fp = outs['fp32']
    N = ro.shape[0]
    rid = trace['ray_id'].long()
    n_c = torch.bincount(rid, minlength=N)
    bad = (fp['ray_stats'][:, 3].long() != n_c)
    assert int(bad.sum()) <= max(1, int(1e-3 * N)) and int(n_c.sum()) > 1000
    shp = shape_info(types.SimpleNamespace(), spec)
    shp.layers = [(w_.double().numpy(), b_.double().numpy()) for w_, b_ in st['rgbnet']]
    x = trace['rgb_feat'].double().numpy()
    assert_exercised(shp.layers, x, act)
    w = trace['weights'].double().numpy()[:, None] * (1 + 1e-4)
    D0 = FEAT_REL * np.abs(x) + 2.0 ** -24
    l_f, E_f = act_logit_bound('fp32', shp, x, None, act, D0=D0, true=True)
    rgb_f = fp['rgb_marched'].double()
    ratios = {}
    for mode, o in outs.items():
        if mode == 'fp32':
            continue
        l_m, E_m = act_logit_bound(mode, shp, x, None, act, D0=D0, true=True)
        Em = np.maximum(E_m, E_f)
        zc = np.clip(0.0, l_f - Em, l_f + Em)
        dmax = sig(zc) * (1 - sig(zc))
        s_hi = sig(l_f + Em)
        B, H = np.zeros((N, 3)), np.zeros((N, 3))
        np.add.at(B, rid.numpy(), w * (dmax * (E_m + E_f) + (2 * SIG_REL + 2 * U) * s_hi))
        np.add.at(H, rid.numpy(), w * s_hi)
        B += 2 * np.maximum(n_c.numpy()[:, None] - 1, 0) * U * H + 2 * U * rgb_f.abs().numpy()
        d = (o['rgb_marched'].double() - rgb_f).abs().numpy()
        keep = ~bad.numpy()
        ok = d[keep] <= B[keep]
        assert ok.all(), (mode, int((~ok).sum()), float((d[keep] / np.maximum(B[keep], 1e-300)).max()))
        ratios[mode] = float((d[keep] / np.maximum(B[keep], 1e-300)).max())
    print(skw, act, 'per-ray error/bound against fp32', {k: f'{v:.3g}' for k, v in ratios.items()})


@pytest.mark.parametrize('act', ACTS)
@pytest.mark.parametrize('regime', ['fog', 'shell'])
def test_ws_against_fp32_per_ray(cuda_device, act, regime):
    """The LLFF shape (configuration 6): ws on image tiles and in flat ray order within the per-ray bound of
    test_gpu_march_mlp.check_per_ray_against_fp32 against fp32 mode, with the activation's error model."""
    from test_gpu_march_mlp import WS_RING_SPECS, check_per_ray_against_fp32, ws_both_orders
    st = make_state('cfgB', xy=48, depth=32, regime=regime)
    x = scale_state_rgbnet(st, act)
    assert_exercised([(W.double().numpy(), b.double().numpy()) for W, b in st['rgbnet']], x, act)
    hw = (40, 52)
    rays, kw = rays_for(st, *hw)
    m = mpi_model(st, act, cuda_device)
    n_c, _ = check_per_ray_against_fp32(m, st, WS_RING_SPECS['cfgB'], rays, kw, ws_both_orders(hw), cuda_device, (act, regime),
                                        act=act)
    assert int(n_c.sum()) > 1000


def test_profiled_kernel_is_relu_only(cuda_device):
    from k4nerf import _lib
    st = make_state('cfgB', xy=16, depth=16, regime='fog')
    m = mpi_model(st, 'gauss', cuda_device)
    (ro, rd, vd), kw = rays_for(st, 8, 8)
    phases = torch.zeros((200, 4, _lib.K4_PHASE_SLOTS), dtype=torch.int64, device=cuda_device)
    with pytest.raises(_lib.K4Error, match='unsupported configuration'):
        m.render_rays(ro.to(cuda_device), rd.to(cuda_device), vd.to(cuda_device), kw, mlp_mode='ws', phases=phases)


# ---------------------------------------------------------------------------------------------------------------------
# 3. at scale
# ---------------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope='module')
def ref_ops(cuda_device):
    from oracle import ops
    if not os.path.exists(ops.ref_ext_path()):
        pytest.skip('oracle/_ref/render_utils_cuda.so not built (needs /root/reference at build time)')
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    return ops.RefExtOps()


def psnr_floor(st, act, n=20000):
    """rgb PSNR floor of ws against the fp32 reference, fixed before the run from the per-sample bound: per ray both
    colours lie within sum_i w_i sigma'_max E_i of the fp64 model's (sum w <= 1, sigma' <= 1/4), so
    |ours - ref| <= (E_ws + E_fp32) / 4 at the largest E over n inputs drawn from the scene's grids
    (mpi_act.sample_inputs), inflated 4x for the samples not drawn; PSNR >= -20 log10 of that.  Capped at the 70 dB bar
    of the relu scale tests (test_gpu_scale.py), which also absorbs borderline-sample flips."""
    spec = ('scale', 'cfgB', 9, 0, 0, 64, 1, 6)
    shp = shape_info(types.SimpleNamespace(), spec)
    shp.layers = [(w_.double().numpy(), b_.double().numpy()) for w_, b_ in st['rgbnet']]
    x = mpi_act.sample_inputs(st, n, seed=1)
    D0 = FEAT_REL * np.abs(x) + 2.0 ** -24
    _, E_w = act_logit_bound('ws', shp, x, None, act, D0=D0, true=True)
    _, E_f = act_logit_bound('fp32', shp, x, None, act, D0=D0, true=True)
    err = float((E_w + E_f).max())                  # (E_ws + E_fp32) / 4, inflated 4x
    return min(70.0, -20 * math.log10(err)), x, shp


@pytest.mark.parametrize('act', ACTS)
def test_mpi_384x384x256_at_1008x756(ref_ops, cuda_device, act):
    from oracle import pipeline, scenes
    from test_gpu_scale import check_against_gpu_oracle
    st = make_state('cfgB', xy=384, depth=256, regime='fog')
    scale_state_rgbnet(st, act)
    bar, x, shp = psnr_floor(st, act)
    assert_exercised(shp.layers, x, act)
    dev = cuda_device
    ro, rd, vd = [t.to(dev) for t in scenes.llff_rays(756, 1008)]
    kw = dict(scenes.RENDER_KW_MPI)
    st_dev = pipeline.state_to(st, dev)
    with oracle_act(act):
        ref, stats = ref_forward_chunked(st_dev, ro, rd, vd, kw, ref_ops, chunk=8192)
    del st_dev
    m = mpi_model(st, act, dev)
    assert m.resolve_mlp_mode('auto') == 'ws'
    ours = m.render_rays(ro, rd, vd, kw, image_hw=(756, 1008), mlp_mode='ws', debug=True)
    torch.cuda.synchronize()
    cmp = check_against_gpu_oracle(ours, ref, stats, ro.shape[0], f'cfgB-384x384x256-1008x756-fog-{act}', rgb_bar=bar)
    assert torch.equal(ours['alphainv_last'], ref['alphainv_last'].to(dev)) or \
        int((ours['alphainv_last'] != ref['alphainv_last'].to(dev)).sum()) <= max(1, int(1e-4 * ro.shape[0]))
    print(act, 'PSNR floor', round(bar, 1), 'dB, measured', cmp)


# ---------------------------------------------------------------------------------------------------------------------
# 4. end to end
# ---------------------------------------------------------------------------------------------------------------------
def test_gauss_checkpoint_load_model_render_viewpoints_and_autograd(cuda_device, tmp_path):
    from oracle import ops, pipeline, scenes
    from k4nerf import dmpigo, render, train_forward, utils
    dev = cuda_device
    st = make_state('cfgB', xy=40, depth=24, regime='fog')
    scale_state_rgbnet(st, 'gauss')
    m0 = mpi_model(st, 'gauss')
    path = tmp_path / 'fine_last.tar'
    torch.save({'global_step': 0, 'model_kwargs': m0.get_kwargs(), 'model_state_dict': m0.state_dict()}, path)
    m = utils.load_model(dmpigo.DirectMPIGO, str(path)).to(dev)
    assert m.act_type == 'gauss'
    H, W = 24, 32
    K, c2w = scenes.llff_camera(H, W, (0.05, -0.03, 0.0))
    kw = dict(scenes.RENDER_KW_MPI)
    rgbs, depths, _, _, _, _ = render.render_viewpoints(m, np.array([c2w.numpy()]), np.array([[H, W]]), np.array([K]), True, kw)
    ro, rd, vd = pipeline.get_rays_of_a_view(H, W, K, c2w, ndc=True, inverse_y=False, flip_x=False, flip_y=False)
    ro, rd, vd = [t.reshape(-1, 3).contiguous() for t in (ro, rd, vd)]
    with oracle_act('gauss'):
        ref = pipeline.forward(st, ro, rd, vd, ops.CpuOps, **kw)
    frame = torch.from_numpy(rgbs[0]).reshape(-1, 3).double()
    p = pipeline.psnr(frame, ref['rgb_marched'].double())
    assert p >= 50.0, p
    # forward under autograd: the materialised pipeline (train_forward) evaluates m.rgbnet with the shared Gaussian
    m.k0.grid.requires_grad_(True)
    out = m(ro.to(dev), rd.to(dev), vd.to(dev), **kw)
    assert 'weights' in out and out['rgb_marched'].requires_grad
    out['rgb_marched'].sum().backward()
    assert torch.isfinite(m.k0.grid.grad).all() and float(m.k0.grid.grad.abs().sum()) > 0
    with torch.no_grad():
        fused = m.render_rays(ro.to(dev), rd.to(dev), vd.to(dev), kw, mlp_mode='ws', debug=True)
        unfused = train_forward.forward_samples(m, ro.to(dev), rd.to(dev), vd.to(dev), **kw)
    torch.cuda.synchronize()
    assert torch.equal(fused['alphainv_last'], unfused['alphainv_last'])
    # per ray within the per-sample bound of ws against fp32, summed with the sample weights (sum w <= 1, sigma' <= 1/4)
    spec = ('e2e', 'cfgB', 9, 0, 0, 64, 1, 6)
    shp = shape_info(types.SimpleNamespace(), spec)
    shp.layers = [(w_.double().numpy(), b_.double().numpy()) for w_, b_ in st['rgbnet']]
    x = mpi_act.sample_inputs(st, 20000, seed=2)
    D0 = FEAT_REL * np.abs(x) + 2.0 ** -24
    _, E_w = act_logit_bound('ws', shp, x, None, 'gauss', D0=D0, true=True)
    _, E_f = act_logit_bound('fp32', shp, x, None, 'gauss', D0=D0, true=True)
    bound = float((E_w + E_f).max())          # 4x the sigma' bound: room for the samples not drawn
    d = (fused['rgb_marched'] - unfused['rgb_marched']).abs().max().item()
    assert d <= bound, (d, bound)
    print('end to end: render_viewpoints PSNR', round(p, 1), 'dB; fused vs autograd forward', d, 'bound', bound)
