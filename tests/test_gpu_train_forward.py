"""GPU: the training-side forward (k4nerf/train_forward.py, SURVEY.md section 8 f-2).

(i) values: the per-sample lists and per-ray outputs against the oracle pipeline running on the
reference's own kernels (oracle/_ref) on the same device; (ii) a few MaskedAdam steps reduce the loss.
The gradients are tested against a float64 restatement in test_gpu_train_grad.py."""
import os

import pytest
import torch

import k4nerf
from k4nerf import train_forward
from helpers import make_state, model_from_state, rays_for
from oracle import ops, pipeline

pytestmark = pytest.mark.gpu


@pytest.fixture(scope='module')
def ref_ops(cuda_device):
    if not os.path.exists(os.path.join(os.path.dirname(ops.ref_ext_path()), 'ub360_utils_cuda.so')):
        pytest.skip('oracle/_ref not built')
    return ops.RefExtOps()


def _state(name, regime):
    if name == 'cfgB':
        return make_state(name, xy=40, depth=24, regime=regime)
    return make_state(name, res=32, regime=regime)


@pytest.mark.parametrize('name', ['cfgA', 'cfgB', 'cfgC'])
@pytest.mark.parametrize('regime', ['fog', 'shell'])
def test_sample_lists_match_reference_kernel_pipeline(ref_ops, cuda_device, name, regime):
    dev = cuda_device
    torch.backends.cuda.matmul.allow_tf32 = False
    st = _state(name, regime)
    (ro, rd, vd), kw = rays_for(st, 24, 32, **({'radius': 0.6} if name == 'cfgC' else {}))
    ro, rd, vd = ro.to(dev), rd.to(dev), vd.to(dev)
    ref = pipeline.forward(pipeline.state_to(st, dev), ro, rd, vd, ref_ops, **kw)
    m = model_from_state(st, dev)
    with torch.no_grad():
        ours = train_forward.forward_samples(m, ro, rd, vd, **kw)
    assert ours['ray_id'].shape == ref['ray_id'].shape and torch.equal(ours['ray_id'], ref['ray_id'])
    assert torch.equal(ours['alphainv_last'], ref['alphainv_last'])
    assert torch.equal(ours['weights'], ref['weights']) and torch.equal(ours['raw_alpha'], ref['raw_alpha'])
    assert torch.allclose(ours['raw_rgb'], ref['raw_rgb'], atol=1e-6)
    assert torch.allclose(ours['rgb_marched'], ref['rgb_marched'], atol=1e-5)
    assert torch.allclose(ours['depth'], ref['depth'], atol=1e-5)
    assert ours['rgb_feature'] is ours['rgb_marched']
    if name != 'cfgA':
        assert ours['n_max'] == ref['n_max'] and torch.allclose(ours['s'], ref['s'], atol=1e-7)
    # and the fused inference kernel agrees with its un-fused restatement
    with torch.no_grad():
        fused = m(ro, rd, vd, **kw)
    assert pipeline.psnr(fused['rgb_marched'].cpu(), ours['rgb_marched'].cpu()) > 60


def test_masked_adam_training_steps_reduce_the_loss(cuda_device):
    dev = cuda_device
    st = make_state('cfgA', res=24, regime='fog')
    (ro, rd, vd), kw = rays_for(st, 16, 16)
    ro, rd, vd = ro.to(dev), rd.to(dev), vd.to(dev)
    m = model_from_state(st, dev)
    target = torch.full((ro.shape[0], 3), 0.25, device=dev)
    opt = k4nerf.MaskedAdam([
        {'params': [m.density.grid], 'lr': 0.1, 'skip_zero_grad': True},
        {'params': [m.k0.grid], 'lr': 0.1, 'skip_zero_grad': True},
        {'params': list(m.rgbnet.parameters()), 'lr': 1e-3, 'skip_zero_grad': False}])
    losses = []
    for step in range(8):
        opt.zero_grad(set_to_none=True)
        out = m(ro, rd, vd, global_step=step, **kw)
        loss = ((out['rgb_marched'] - target) ** 2).mean()
        loss.backward()
        m.density_total_variation_add_grad(1e-5, False)
        opt.step()
        losses.append(float(loss.detach()))
        if step in (2, 5):
            # mid-training validation as the reference loop does it (run_sr.py:586-599): NO manual invalidate --
            # the optimiser kernels bump the parameters' versions, so the fused render sees the new weights
            with torch.no_grad():
                fused = m(ro, rd, vd, **kw)['rgb_marched'].clone()
                again = m(ro, rd, vd, **kw)['rgb_marched']
                unfused = train_forward.forward_samples(m, ro, rd, vd, **kw)['rgb_marched']
            assert pipeline.psnr(fused.cpu(), unfused.cpu()) > 55, step
            assert pipeline.psnr(fused.cpu(), again.cpu()) > 90
    assert losses[-1] < 0.9 * losses[0] and all(b < a for a, b in zip(losses, losses[1:])), losses
    with torch.no_grad():                                         # the fused kernel renders the trained scene
        fused = m(ro, rd, vd, **kw)
        unfused = train_forward.forward_samples(m, ro, rd, vd, **kw)
    assert pipeline.psnr(fused['rgb_marched'].cpu(), unfused['rgb_marched'].cpu()) > 55


def test_scene_rebuilds_when_a_baked_scalar_changes(cuda_device):
    """fast_color_thres is baked into the device scene: changing it must change the render."""
    dev = cuda_device
    st = make_state('cfgA', res=24, regime='fog')
    (ro, rd, vd), kw = rays_for(st, 16, 16)
    ro, rd, vd = ro.to(dev), rd.to(dev), vd.to(dev)
    m = model_from_state(st, dev)
    a = m.render_rays(ro, rd, vd, kw, debug=True)['counters'].clone()
    m.fast_color_thres = 0.05
    b = m.render_rays(ro, rd, vd, kw, debug=True)['counters'].clone()
    assert int(b[2]) < int(a[2]), (a, b)                      # fewer shaded samples at the higher threshold


def test_dcvgo_training_keys_and_threshold_schedule(cuda_device):
    """lib/dcvgo.py:358-371 key set (run_sr.py:531-532 reads 't' / 'raw_density') and the dict-valued
    fast_color_thres schedule (lib/dcvgo.py:269-271)."""
    dev = cuda_device
    st = make_state('cfgC', res=24, regime='fog')
    (ro, rd, vd), kw = rays_for(st, 12, 16, radius=0.6)
    ro, rd, vd = ro.to(dev), rd.to(dev), vd.to(dev)
    m = model_from_state(st, dev)
    out = m(ro, rd, vd, global_step=3, is_train=True, **kw)
    n = out['weights'].shape[0]
    for k in ('t', 'raw_density', 'step_id', 's', 'raw_alpha', 'ray_id'):
        assert out[k].shape[0] == n, k
    assert out['wsum_mid'].shape == (ro.shape[0],) and out['n_max'] > 0
    assert torch.allclose(out['s'], 1 - 1 / (1 + out['t']))
    assert (out['wsum_mid'] <= out['weights'].new_zeros(ro.shape[0]).index_add_(0, out['ray_id'], out['weights']) + 1e-6).all()
    # raw_alpha is the activation of raw_density
    interval = float(kw['stepsize'] * m.voxel_size_ratio)
    alpha = 1 - (1 + torch.exp(out['raw_density'].flatten() + float(m.act_shift))) ** (-interval)
    assert torch.allclose(alpha, out['raw_alpha'], atol=1e-6)
    m._fast_color_thres = {0: 1e-4, 5: 0.03}
    m.fast_color_thres = 1e-4
    with torch.no_grad():
        m(ro, rd, vd, global_step=4, **kw)
        assert m.fast_color_thres == 1e-4
        a = m.render_rays(ro, rd, vd, kw, debug=True)['counters'].clone()
        m(ro, rd, vd, global_step=5, **kw)
        assert m.fast_color_thres == 0.03
        b = m.render_rays(ro, rd, vd, kw, debug=True)['counters'].clone()
    assert int(b[2]) < int(a[2])
