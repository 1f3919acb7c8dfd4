"""GPU: the profiled instantiation of the warp-specialised marcher (k4_testing_march_phases) computes what the production
kernel computes, and its phase counters account for every cycle and every batch.

- Outputs: alphainv_last, depth, ray_stats and counters are bit-identical to the production kernel's; rgb agrees within
  2e-5, the bound test_gpu_marcher.py allows two ws runs (the colour atomics of a ray land in a run-dependent order).
- Per CTA and warpgroup, the phases add up to the elapsed cycles.  Each phase boundary charges the cycles since the
  previous one, so the sum is exact up to the stated slack of 1e-6 of the elapsed cycles.
- The batches the MLP groups consume, and those the marchers submit, both equal counters[3].
"""
import pytest
import torch

from helpers import make_state, model_from_state, rays_for

pytestmark = pytest.mark.gpu

SCENES = [('cfgA', dict(res=48, regime='fog'), 240, 320),       # 600 tiles: more than two per marcher group
          ('cfgA', dict(res=48, regime='shell'), 240, 320),
          ('cfgB', dict(xy=48, depth=32, regime='fog'), 96, 128),
          ('cfgC', dict(res=48, regime='fog'), 64, 96)]


def profiled_and_production(dev, name, kw, H, W):
    from k4nerf import _lib
    st = make_state(name, **kw)
    rays, rkw = rays_for(st, H, W)
    m = model_from_state(st, dev)
    ro, rd, vd = [t.to(dev) for t in rays]
    prod = m.render_rays(ro, rd, vd, rkw, image_hw=(H, W), mlp_mode='ws', debug=True)
    ph = torch.zeros((1024, 4, _lib.K4_PHASE_SLOTS), dtype=torch.int64, device=dev)
    prof = m.render_rays(ro, rd, vd, rkw, image_hw=(H, W), mlp_mode='ws', debug=True, phases=ph)
    torch.cuda.synchronize()
    return prod, prof, ph[:prof['n_ctas']].cpu()


@pytest.mark.parametrize('name,kw,H,W', SCENES, ids=[f'{s[0]}-{s[1].get("regime")}' for s in SCENES])
def test_profiled_kernel_outputs_and_phase_accounting(cuda_device, name, kw, H, W):
    from k4nerf import _lib
    prod, prof, ph = profiled_and_production(cuda_device, name, kw, H, W)
    assert torch.equal(prod['alphainv_last'], prof['alphainv_last'])
    assert torch.equal(prod['depth'], prof['depth'])
    assert torch.equal(prod['ray_stats'], prof['ray_stats'])
    assert torch.equal(prod['counters'], prof['counters'])
    assert (prod['rgb_marched'] - prof['rgb_marched']).abs().max().item() <= 2e-5

    n_tiles = ((W + 15) // 16) * ((H + 7) // 8)
    assert 1 <= prof['n_ctas'] <= (n_tiles + 1) // 2
    assert ph.shape == (prof['n_ctas'], 4, _lib.K4_PHASE_SLOTS)
    elapsed = ph[..., 0]
    assert bool((elapsed > 0).all())
    parts = ph[..., 1:_lib.K4_PHASE_SLOTS - 1]
    assert bool((parts >= 0).all())
    slack = elapsed.double() * 1e-6
    assert bool(((parts.sum(-1) - elapsed).abs().double() <= slack).all())
    batches = int(prof['counters'][3])
    assert batches > 0
    assert int(ph[:, 2:, _lib.K4_PHASE_SLOTS - 1].sum()) == batches     # consumed by the MLP groups
    assert int(ph[:, :2, _lib.K4_PHASE_SLOTS - 1].sum()) == batches     # submitted by the marchers


def test_too_few_cta_slots_is_an_argument_error(cuda_device):
    """A phase buffer too small for the launch is reported, and nothing runs."""
    from k4nerf import _lib
    st = make_state('cfgA', res=32, regime='fog')
    rays, rkw = rays_for(st, 64, 64)                                    # 32 tiles -> 16 CTAs
    m = model_from_state(st, cuda_device)
    ro, rd, vd = [t.to(cuda_device) for t in rays]
    ph = torch.zeros((15, 4, _lib.K4_PHASE_SLOTS), dtype=torch.int64, device=cuda_device)
    with pytest.raises(_lib.K4Error, match='invalid'):
        m.render_rays(ro, rd, vd, rkw, image_hw=(64, 64), mlp_mode='ws', phases=ph)
    ph = torch.zeros((16, 4, _lib.K4_PHASE_SLOTS), dtype=torch.int64, device=cuda_device)
    assert m.render_rays(ro, rd, vd, rkw, image_hw=(64, 64), mlp_mode='ws', phases=ph)['n_ctas'] == 16
