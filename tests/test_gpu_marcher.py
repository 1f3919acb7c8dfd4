"""GPU parity tests proper: the fused sm_90a marcher (through the C ABI) against the CPU oracle on
the same seeded scenes.

Bars (north_star): geometric quantities bit-exact -- t_min/t_max, per-ray step counts, number of
in-box samples (S_m) and of occupancy hits (S_d); value-dependent survivors (S_c: alpha/weight
thresholds, T < 1e-3 early-out) may flip on borderline samples because expf/powf differ by <= 2 ulp
between the CUDA math library and the host libm -- flip rate must stay below 1e-4; rendered values
within PSNR >= 70 dB of the oracle (fp32 / f16x3 modes; MSE <= 1e-7, i.e. dPSNR << 0.01 dB on any
render of 20-40 dB), >= 55 dB for the single-pass f16 tensor-core mode.
"""
import pytest
import torch

from oracle import ops, pipeline
from helpers import compare, make_state, model_from_state, rays_for

pytestmark = pytest.mark.gpu

PSNR_BAR = {'fp32': 80.0, 'f16x3': 70.0, 'f16': 70.0, 'ws': 70.0}


def run_both(st, rays, kw, dev, mode, image_hw=None):
    ro, rd, vd = rays
    stats = {}
    ref = pipeline.forward(st, ro, rd, vd, ops.CpuOps, stats=stats, **kw)
    m = model_from_state(st, dev)
    ours = m.render_rays(ro.to(dev), rd.to(dev), vd.to(dev), kw, image_hw=image_hw, mlp_mode=mode, debug=True)
    torch.cuda.synchronize()
    return ours, ref, stats


def check_geometry(ours, ref, stats, st, n):
    """Bit-exact geometry: per-ray step counts, t_min/t_max, and per-ray numbers of in-box samples
    and occupancy hits visited before the transmittance early-out.  The early-out itself
    (T < 1e-3) and the threshold survivors are value dependent (expf/powf differ by <= 2 ulp between
    the CUDA math library and the host libm), so a ray whose T lands within rounding of 1e-3 may stop
    one sample apart: at most 1e-4 of the rays / samples may differ."""
    c = ours['counters'].cpu().tolist()
    rs = ours['ray_stats'].cpu().long()
    ors = ref['_ray_stats'].cpu()
    bad = (rs[:, 1] != ors[:, 0]) | (rs[:, 2] != ors[:, 1])
    assert int(bad.sum()) <= max(1, int(1e-4 * n)), ('rays with different S_m/S_d', int(bad.sum()), n)
    assert abs(c[0] - stats['S_m']) <= max(300, 1e-4 * stats['S_m']), ('S_m', c[0], stats['S_m'])
    assert abs(c[1] - stats['S_d']) <= max(300, 1e-4 * stats['S_d']), ('S_d', c[1], stats['S_d'])
    assert abs(c[2] - stats['S_c']) <= max(2, 1e-4 * stats['S_c']), ('S_c', c[2], stats['S_c'])
    assert int(rs[:, 1].sum()) == c[0] and int(rs[:, 2].sum()) == c[1] and int(rs[:, 3].sum()) == c[2]
    if st['kind'] == 'dvgo':
        assert torch.equal(rs[:, 0], ref['_N_steps'].cpu()), 'per-ray step counts differ'
        tm = ours['t_minmax'].cpu()
        assert torch.equal(tm[:, 0], ref['_t_min'].cpu()) and torch.equal(tm[:, 1], ref['_t_max'].cpu()), 't_min/t_max not bit-exact'


@pytest.mark.parametrize('regime', ['fog', 'shell'])
@pytest.mark.parametrize('mode', ['fp32', 'f16x3', 'f16', 'ws'])
def test_cfgA_parity(cuda_device, regime, mode):
    st = make_state('cfgA', res=48, regime=regime)
    rays, kw = rays_for(st, 40, 52)
    ours, ref, stats = run_both(st, rays, kw, cuda_device, mode)
    n = rays[0].shape[0]
    check_geometry(ours, ref, stats, st, n)
    cmp = compare(ours, ref, n)
    assert cmp['rgb_marched_psnr'] >= PSNR_BAR[mode], cmp
    assert cmp['alphainv_last_maxabs'] <= 2e-5, cmp
    assert cmp['depth_maxabs'] <= 2e-5, cmp


@pytest.mark.parametrize('mode', ['fp32', 'f16x3', 'ws'])
def test_cfgA_2d_tiles_equal_linear_order(cuda_device, mode):
    """8x4 pixel-tile scheduling must not change any ray's result."""
    st = make_state('cfgA', res=32, regime='shell')
    rays, kw = rays_for(st, 37, 45)
    dev = cuda_device
    m = model_from_state(st, dev)
    ro, rd, vd = [t.to(dev) for t in rays]
    a = m.render_rays(ro, rd, vd, kw, mlp_mode=mode)
    b = m.render_rays(ro, rd, vd, kw, image_hw=(37, 45), mlp_mode=mode)
    assert torch.equal(a['alphainv_last'], b['alphainv_last'])
    assert torch.equal(a['depth'], b['depth'])
    if mode == 'fp32':
        assert torch.equal(a['rgb_marched'], b['rgb_marched'])
    else:
        assert (a['rgb_marched'] - b['rgb_marched']).abs().max().item() < (1e-5 if mode != 'ws' else 2e-5)


def test_cfgA_not_direct_and_width64(cuda_device):
    """rgbnet_direct=False (diffuse term, lib/dvgo.py:385-386,412) and a 64-wide MLP."""
    for mode in ('fp32', 'f16x3', 'f16'):
        st = make_state('cfgA', res=32, regime='fog', rgbnet_direct=False, width=64)
        rays, kw = rays_for(st, 24, 24)
        ours, ref, stats = run_both(st, rays, kw, cuda_device, mode)
        check_geometry(ours, ref, stats, st, rays[0].shape[0])
        cmp = compare(ours, ref, rays[0].shape[0])
        assert cmp['rgb_marched_psnr'] >= PSNR_BAR[mode], (mode, cmp)


def test_cfg1_colour_grid_no_mlp(cuda_device):
    """BASELINE.json configs[0]: coarse-stage shape, rgb = sigmoid(k0), no MLP."""
    st = make_state('cfg1', res=32)
    rays, kw = rays_for(st, 64, 64)
    ours, ref, stats = run_both(st, rays, kw, cuda_device, 'fp32')
    check_geometry(ours, ref, stats, st, rays[0].shape[0])
    cmp = compare(ours, ref, rays[0].shape[0])
    assert cmp['rgb_marched_psnr'] >= 80.0, cmp


@pytest.mark.parametrize('regime', ['fog', 'shell'])
@pytest.mark.parametrize('mode', ['fp32', 'f16x3', 'f16', 'ws'])
def test_cfgB_mpi_parity(cuda_device, regime, mode):
    st = make_state('cfgB', xy=48, depth=32, regime=regime)
    rays, kw = rays_for(st, 30, 40)
    ours, ref, stats = run_both(st, rays, kw, cuda_device, mode)
    n = rays[0].shape[0]
    check_geometry(ours, ref, stats, st, n)
    cmp = compare(ours, ref, n)
    assert cmp['rgb_marched_psnr'] >= PSNR_BAR[mode], cmp
    assert cmp['alphainv_last_maxabs'] <= 2e-5, cmp


def test_cfgB_positional_encodings(cuda_device):
    st = make_state('cfgB', xy=32, depth=16, regime='fog', viewbase_pe=2, spatial_pe=3)
    rays, kw = rays_for(st, 16, 20)
    for mode in ('fp32', 'f16x3'):
        ours, ref, stats = run_both(st, rays, kw, cuda_device, mode)
        cmp = compare(ours, ref, rays[0].shape[0])
        assert cmp['rgb_marched_psnr'] >= PSNR_BAR[mode], (mode, cmp)


def test_edge_cases(cuda_device):
    dev = cuda_device
    st = make_state('cfgA', res=24, regime='fog')
    m = model_from_state(st, dev)
    kw = rays_for(st, 4, 4)[1]
    # empty batch
    e = torch.zeros(0, 3, device=dev)
    with torch.no_grad():                      # inference: the fused kernel (autograd on -> train_forward)
        out = m(e, e, e, **kw)
    assert out['rgb_marched'].shape == (0, 3) and out['rgb_feature'] is out['rgb_marched']
    # rays that miss the box, axis-parallel rays (zero components -> the 1e-6 substitution), ragged N
    ro = torch.tensor([[0, 0, 4.], [5, 5, 5.], [0.3, -0.2, 4.], [0, 0, 0.]])
    rd = torch.tensor([[0, 0, -1.], [1, 0, 0.], [0, 0, -2.], [0, 1, 0.]])
    vd = rd / rd.norm(dim=-1, keepdim=True)
    ro, rd, vd = ro.repeat(9, 1)[:33], rd.repeat(9, 1)[:33], vd.repeat(9, 1)[:33]
    stats = {}
    ref = pipeline.forward(st, ro, rd, vd, ops.CpuOps, stats=stats, **kw)
    for mode in ('fp32', 'f16x3', 'ws'):
        ours = m.render_rays(ro.to(dev), rd.to(dev), vd.to(dev), kw, mlp_mode=mode, debug=True)
        check_geometry(ours, ref, stats, st, 33)
        cmp = compare(ours, ref, 33)
        assert cmp['rgb_marched_maxabs'] < (1e-4 if mode != 'ws' else 5e-3), (mode, cmp)
        assert torch.equal(ours['alphainv_last'][1].cpu(), torch.tensor(1.0))   # missed the box: T stays 1


def test_forward_contract_and_scene_refresh(cuda_device):
    dev = cuda_device
    st = make_state('cfgA', res=24, regime='fog')
    m = model_from_state(st, dev)
    (ro, rd, vd), kw = rays_for(st, 8, 8)
    with torch.no_grad():
        out = m(ro.to(dev), rd.to(dev), vd.to(dev), **kw)
    assert set(out) >= {'rgb_marched', 'rgb_feature', 'alphainv_last', 'depth'} and 'weights' not in out
    assert out['rgb_feature'].data_ptr() == out['rgb_marched'].data_ptr()     # the reference's alias
    kw2 = dict(kw); kw2['render_depth'] = False
    with torch.no_grad():
        assert 'depth' not in m(ro.to(dev), rd.to(dev), vd.to(dev), **kw2)
    # in-place parameter edits must invalidate the cached device scene
    before = out['rgb_marched'].clone()
    with torch.no_grad():
        m.density.grid.add_(3.0)
        after = m(ro.to(dev), rd.to(dev), vd.to(dev), **kw)['rgb_marched']
    assert (after - before).abs().max().item() > 1e-3


def test_make_rays_matches_reference_formulas(cuda_device):
    import k4nerf
    from oracle import scenes
    for ndc in (False, True):
        H, W = 21, 34
        K, c2w = (scenes.llff_camera(H, W, (0.05, -0.03, 0.0)) if ndc else scenes.blender_camera(H, W))
        for inverse_y, fx, fy in ((False, False, False), (True, True, False), (False, False, True)):
            ref = pipeline.get_rays_of_a_view(H, W, K, c2w, ndc, inverse_y, fx, fy)
            got = k4nerf.get_rays_of_a_view(H, W, K, c2w.to(cuda_device), ndc, inverse_y, fx, fy)
            for a, b in zip(got, ref):
                assert (a.cpu() - b).abs().max().item() <= 2e-6 * max(1.0, b.abs().max().item())


# (the persistent multi-tile case lives in test_gpu_scale.py::test_persistent_multi_tile_vs_gpu_oracle, against the
# reference kernels' pipeline instead of the repo's own mma.sync kernel)


# ---------------------------------------------------------------------------------------------------------------
# wgmma marcher for every shape the reference can produce (csrc/k4_ws_cfgs.h): exact instantiations and models that
# run zero-padded on a larger instantiation.  `auto` must resolve to `ws` for all of them.
# ---------------------------------------------------------------------------------------------------------------
WS_SHAPES = [
    # kind, scene kwargs, expected config id (k4_ws_cfgs.h)
    ('cfgA', dict(k0_dim=12, viewbase_pe=0, width=128), 0),                       # configs/syn/1x_chair_joint_l1+gan.py
    ('cfgA', dict(k0_dim=12, viewbase_pe=4, width=64), 3),
    ('cfgA', dict(k0_dim=12, viewbase_pe=0, width=64), 2),
    ('cfgA', dict(k0_dim=12, viewbase_pe=4, width=128, rgbnet_direct=False), 4),  # diffuse term, odd feature count (9)
    ('cfgA', dict(k0_dim=15, viewbase_pe=4, width=128, rgbnet_direct=False), 4),
    ('cfgA', dict(k0_dim=6, viewbase_pe=3, width=96), 1),                         # padded: fewer channels / frequencies / units
    ('cfgA', dict(k0_dim=9, viewbase_pe=2, width=64), 3),
    ('cfgA', dict(k0_dim=16, viewbase_pe=6, width=128), 5),
    ('cfgA', dict(k0_dim=7, viewbase_pe=2, width=40, rgbnet_direct=False), 4),
    ('cfgB', dict(k0_dim=12, viewbase_pe=4, spatial_pe=0, width=128), 7),
    ('cfgB', dict(k0_dim=9, viewbase_pe=2, spatial_pe=3, width=64), 8),           # lib/dmpigo.py:96-100 position code
    ('cfgB', dict(k0_dim=12, viewbase_pe=4, spatial_pe=5, width=128), 8),
    ('cfgC', dict(k0_dim=12, viewbase_pe=0, width=128), 9),
    ('cfgC', dict(k0_dim=8, viewbase_pe=2, width=64), 10),
]


@pytest.mark.parametrize('kind,skw,cfg_id', WS_SHAPES, ids=[f'{k}-{"-".join(f"{a}{b}" for a, b in v.items())}' for k, v, _ in WS_SHAPES])
def test_tcgen05_marcher_covers_other_shapes(cuda_device, kind, skw, cfg_id):
    from k4nerf import _lib
    dev = cuda_device
    if kind == 'cfgB':
        st = make_state(kind, xy=40, depth=24, regime='fog', **skw)
        hw = (24, 32)
    else:
        st = make_state(kind, res=40, regime='fog', **skw)
        hw = (32, 40)
    rays, kw = rays_for(st, *hw, **({'radius': 0.6} if kind == 'cfgC' else {}))
    ro, rd, vd = rays
    stats = {}
    ref = pipeline.forward(st, ro, rd, vd, ops.CpuOps, stats=stats, **kw)
    m = model_from_state(st, dev)
    assert m.resolve_mlp_mode('auto') == 'ws'
    assert _lib.lib.k4_scene_ws_config(m._get_scene().ptr) == cfg_id
    n = ro.shape[0]
    for img in (hw, None):
        ours = m.render_rays(ro.to(dev), rd.to(dev), vd.to(dev), kw, image_hw=img, mlp_mode='auto', debug=True)
        torch.cuda.synchronize()
        check_geometry(ours, ref, stats, st, n)
        cmp = compare(ours, ref, n)
        assert cmp['rgb_marched_psnr'] >= PSNR_BAR['ws'], (skw, cmp)
        assert cmp['alphainv_last_maxabs'] <= 2e-5, (skw, cmp)
    # and against the exact-precision kernel on the same device
    exact = m.render_rays(ro.to(dev), rd.to(dev), vd.to(dev), kw, mlp_mode='fp32')
    assert torch.equal(exact['alphainv_last'], ours['alphainv_last'])
    assert (exact['rgb_marched'] - ours['rgb_marched']).abs().max().item() < 5e-3


def test_deeper_mlp_falls_back_to_exact_kernels(cuda_device):
    """rgbnet_depth != 3 has no tensor-core build: auto must pick the fp32 kernel, not fail."""
    st = make_state('cfgA', res=24, regime='fog', depth=4)
    (ro, rd, vd), kw = rays_for(st, 12, 12)
    m = model_from_state(st, cuda_device)
    assert m.resolve_mlp_mode('auto') == 'fp32'
    ref = pipeline.forward(st, ro, rd, vd, ops.CpuOps, **kw)
    ours = m.render_rays(ro.to(cuda_device), rd.to(cuda_device), vd.to(cuda_device), kw)
    assert compare(ours, ref, ro.shape[0])['rgb_marched_psnr'] >= 80.0


# ---------------------------------------------------------------------------------------------------------------
# empty-space skipping is result preserving: same per-ray visit counts, depth, transmittance as the step-by-step walk
# ---------------------------------------------------------------------------------------------------------------
def _blob_state(kind, seed=0):
    """Random sparse occupancy (blobs), density low outside: many skip / no-skip transitions along every ray."""
    import torch.nn.functional as F
    st = make_state('cfgB', xy=56, depth=40, regime='fog') if kind == 'cfgB' else make_state('cfgA', res=64, regime='fog')
    g = torch.Generator().manual_seed(seed)
    ws = list(st['density'].shape[2:])
    seeds = (torch.rand(ws, generator=g) > 0.9985).float()[None, None]
    blobs = F.max_pool3d(seeds, kernel_size=5, stride=1, padding=2)[0, 0] > 0
    st['density'] = torch.where(blobs, torch.full(ws, 3.0), torch.full(ws, -6.0))[None, None].contiguous()
    st['mask_cache'] = pipeline.mask_grid_state(blobs, st['xyz_min'], st['xyz_max'])
    return st


@pytest.mark.parametrize('kind,regime', [('cfgA', 'shell'), ('cfgA', 'blobs'), ('cfgA', 'fog'), ('cfgB', 'shell'), ('cfgB', 'blobs')])
def test_empty_space_skipping_preserves_results(cuda_device, kind, regime, monkeypatch):
    dev = cuda_device
    if regime == 'blobs':
        st = _blob_state(kind)
    else:
        st = make_state(kind, xy=56, depth=40, regime=regime) if kind == 'cfgB' else make_state(kind, res=64, regime=regime)
    (ro, rd, vd), kw = rays_for(st, 96, 128)
    ro, rd, vd = ro.to(dev), rd.to(dev), vd.to(dev)
    stats = {}
    ref = pipeline.forward(st, ro.cpu(), rd.cpu(), vd.cpu(), ops.CpuOps, stats=stats, **kw)
    outs = {}
    for skip in (True, False):
        if skip:
            monkeypatch.delenv('K4_NO_SKIP', raising=False)
        else:
            monkeypatch.setenv('K4_NO_SKIP', '1')          # read by k4_scene_create
        m = model_from_state(st, dev)
        for mode in ('ws', 'f16', 'fp32'):
            for img in ((96, 128), None):
                outs[(skip, mode, img)] = m.render_rays(ro, rd, vd, kw, image_hw=img, mlp_mode=mode, debug=True)
        torch.cuda.synchronize()
    for mode in ('ws', 'f16', 'fp32'):
        for img in ((96, 128), None):
            a, b = outs[(True, mode, img)], outs[(False, mode, img)]
            assert torch.equal(a['ray_stats'], b['ray_stats']), (mode, img)
            assert torch.equal(a['counters'][:3], b['counters'][:3]), (mode, img)
            assert torch.equal(a['alphainv_last'], b['alphainv_last']) and torch.equal(a['depth'], b['depth']), (mode, img)
            if mode == 'fp32':
                assert torch.equal(a['rgb_marched'], b['rgb_marched'])
            else:
                assert (a['rgb_marched'] - b['rgb_marched']).abs().max().item() < 3e-5
    check_geometry(outs[(True, 'ws', (96, 128))], ref, stats, st, ro.shape[0])


@pytest.mark.parametrize('mode', ['f16x3', 'ws', 'fp32'])
def test_render_rays_frames_assembles_the_block_cyclic_frame(cuda_device, mode):
    """k4_render_rays_frames: every rank's rows (8-row blocks dealt round-robin) stored by the kernel straight into the
    image-order frames -- here three 'ranks' one after the other on one GPU, two destination frames each (on a multi-GPU
    node the second one is a peer's frame reached over NVLink).  The assembled frame equals the one-launch frame."""
    from k4nerf import dist as kdist
    st = make_state('cfgA', res=48, regime='fog')
    H, W, world = 50, 72, 3                       # 7 blocks: ranks get 3 / 2 / 2 blocks, the last block is 2 rows
    rays, kw = rays_for(st, H, W)
    kw = dict(kw); kw['render_depth'] = True
    m = model_from_state(st, cuda_device)
    ro, rd, vd = [t.to(cuda_device) for t in rays]
    ref = m.render_rays(ro, rd, vd, kw, image_hw=(H, W), mlp_mode=mode)
    n_full = world * kdist.cyclic_pad_rows(H, world) * W
    frames = [torch.full((5 * n_full,), -3.0, device=cuda_device) for _ in range(2)]
    for rank in range(world):
        rows = kdist.cyclic_rows(H, rank, world).to(cuda_device)
        sel = lambda t: t.view(H, W, 3)[rows].reshape(-1, 3).contiguous()
        tgt = kdist.FrameTarget([f.data_ptr() for f in frames], rank, world, W, n_full)
        hw = (rows.numel(), W) if rank != 1 else None            # rank 1: the linear (no image tiles) ray order
        m.render_rays(sel(ro), sel(rd), sel(vd), kw, image_hw=hw, mlp_mode=mode, out=tgt)
    torch.cuda.synchronize()
    assert torch.equal(frames[0], frames[1])
    got = kdist.frame_views(frames[0], H, W, n_full)
    exact = mode in ('f16x3', 'fp32')              # the wgmma kernels composite with shared-memory atomics: order-dependent rounding
    for k in ('rgb_marched', 'depth', 'alphainv_last'):
        if exact:
            assert torch.equal(got[k], ref[k]), k
        else:
            assert torch.allclose(got[k], ref[k], rtol=0, atol=2e-5), (k, (got[k] - ref[k]).abs().max().item())
    # nothing outside the image rows was touched
    assert bool((frames[0][3 * H * W:3 * n_full] == -3.0).all()) and bool((frames[0][3 * n_full + H * W:4 * n_full] == -3.0).all())
