"""CPU: host-side mirror of the reference API -- constructor arithmetic, state-dict layout,
checkpoint round trip, error behaviour (no compute calls, no GPU)."""
import os
import tempfile

import pytest
import torch

import k4nerf
from oracle import pipeline
from helpers import make_state, model_from_state


def test_dvgo_constructor_matches_oracle_arithmetic():
    st = pipeline.dvgo_state([-1.1, -0.9, -1.0], [1.0, 1.2, 0.8], num_voxels=50 ** 3, num_voxels_base=40 ** 3,
                             alpha_init=1e-2, fast_color_thres=1e-4, rgbnet_dim=12, rgbnet_direct=True)
    m = k4nerf.DirectVoxGO([-1.1, -0.9, -1.0], [1.0, 1.2, 0.8], num_voxels=50 ** 3, num_voxels_base=40 ** 3,
                           alpha_init=1e-2, fast_color_thres=1e-4, rgbnet_dim=12, rgbnet_direct=True)
    assert m.world_size.tolist() == st['world_size'].tolist()
    assert torch.equal(m.voxel_size, st['voxel_size'])
    assert torch.equal(m.voxel_size_ratio, st['voxel_size_ratio'])
    assert torch.equal(m.act_shift, st['act_shift'])
    assert torch.equal(m.mask_cache.xyz2ijk_scale, st['mask_cache']['xyz2ijk_scale'])
    assert torch.equal(m.mask_cache.xyz2ijk_shift, st['mask_cache']['xyz2ijk_shift'])
    assert m.dim0 == st['dim0'] == 39
    assert list(m.density.grid.shape) == list(st['density'].shape)
    assert list(m.k0.grid.shape) == list(st['k0'].shape)


def test_dmpigo_constructor_matches_oracle_arithmetic():
    args = dict(num_voxels=96 * 96 * 64, mpi_depth=64, fast_color_thres=1 / 64 / 5, rgbnet_dim=9, rgbnet_width=64)
    st = pipeline.dmpigo_state([-1.5, -1.67, -1], [1.5, 1.67, 1], **args)
    m = k4nerf.DirectMPIGO([-1.5, -1.67, -1], [1.5, 1.67, 1], act_type='relu', mode_type='mlp', **args)
    assert m.world_size.tolist() == st['world_size'].tolist()
    assert m.voxel_size_ratio == st['voxel_size_ratio']
    assert torch.equal(m.act_shift.grid, st['act_shift_grid'])
    assert m.dim0 == st['dim0'] == 15


def test_state_dict_keys_follow_reference_module_tree():
    m = k4nerf.DirectVoxGO([-1, -1, -1], [1, 1, 1], num_voxels=16 ** 3, num_voxels_base=16 ** 3, alpha_init=1e-2,
                           fast_color_thres=1e-4, rgbnet_dim=12, rgbnet_direct=True, rgbnet_depth=3)
    keys = set(m.state_dict())
    # lib/dvgo.py:116-123: Sequential(Linear, ReLU, Sequential(Linear, ReLU), Linear)
    for k in ('density.grid', 'k0.grid', 'mask_cache.mask', 'mask_cache.xyz2ijk_scale', 'mask_cache.xyz2ijk_shift',
              'act_shift', 'xyz_min', 'xyz_max', 'viewfreq', 'rgbnet.0.weight', 'rgbnet.2.0.weight', 'rgbnet.3.bias',
              'density.xyz_min', 'k0.xyz_max'):
        assert k in keys, k


def test_checkpoint_round_trip_reference_layout():
    st = make_state('cfgA', res=12)
    m = model_from_state(st)
    with tempfile.TemporaryDirectory() as d:
        path = os.path.join(d, 'fine_last.tar')
        # the reference's checkpoint layout, run_sr.py:1163-1168
        torch.save({'global_step': 7, 'model_kwargs': m.get_kwargs(), 'model_state_dict': m.state_dict(),
                    'optimizer_state_dict': {}}, path)
        m2 = k4nerf.utils.load_model(k4nerf.DirectVoxGO, path)
    for k, v in m.state_dict().items():
        assert torch.equal(v, m2.state_dict()[k]), k


def test_load_state_dict_adopts_checkpoint_grid_shapes():
    m = k4nerf.DirectVoxGO([-1, -1, -1], [1, 1, 1], num_voxels=16 ** 3, num_voxels_base=16 ** 3, alpha_init=1e-2,
                           fast_color_thres=1e-4, rgbnet_dim=12, rgbnet_direct=True)
    sd = m.state_dict()
    sd['density.grid'] = torch.zeros(1, 1, 15, 17, 16)
    sd['k0.grid'] = torch.zeros(1, 12, 15, 17, 16)
    sd['mask_cache.mask'] = torch.ones(15, 17, 16, dtype=torch.bool)
    m.load_state_dict(sd)
    assert list(m.k0.grid.shape) == [1, 12, 15, 17, 16]


def test_cpu_tensors_raise_like_check_cuda():
    st = make_state('cfgA', res=8)
    m = model_from_state(st)
    ro = torch.zeros(4, 3)
    with pytest.raises(RuntimeError, match='CUDA'):
        m(ro, ro + 1, ro + 1, near=0.2, far=6, bg=1, stepsize=0.5, render_depth=True)


def test_unsupported_grid_type_raises():
    with pytest.raises(NotImplementedError):
        k4nerf.DirectVoxGO([-1, -1, -1], [1, 1, 1], num_voxels=8 ** 3, num_voxels_base=8 ** 3, alpha_init=1e-2,
                           density_type='TensoRFGrid')


def test_sftnet_state_dict_matches_reference_names():
    from oracle import sftnet
    n = k4nerf.SFTNet(3, 4, 64, 5, 32, 1)
    sd = sftnet.random_state_dict(seed=3)           # names/shapes restated from lib/sr_esrnet.py:411-444
    assert set(n.state_dict()) == set(sd)
    for k, v in n.state_dict().items():
        assert tuple(v.shape) == tuple(sd[k].shape), k
    assert len(n._ordered_convs()) == 229            # SURVEY.md section 2.2: 229 convs per forward
    with pytest.raises(NotImplementedError):
        k4nerf.SFTNet(3, 2, 64, 5, 32, 1)


def test_dcvgo_constructor_contract():
    """DirectContractedVoxGO: buffers, derived sizes, checkpoint keys and the step list follow
    lib/dcvgo.py:27-160,239-248."""
    import numpy as np
    m = k4nerf.DirectContractedVoxGO(xyz_min=[-2, -1, 0], xyz_max=[2, 3, 4], num_voxels=40 ** 3, num_voxels_base=40 ** 3,
                                     alpha_init=1e-2, fast_color_thres=1e-4, bg_len=0.2, rgbnet_dim=12,
                                     rgbnet_depth=3, rgbnet_width=128, viewbase_pe=4)
    assert torch.equal(m.scene_center, torch.tensor([0., 1., 2.])) and torch.equal(m.scene_radius, torch.tensor([2., 2., 2.]))
    assert torch.allclose(m.xyz_min, torch.tensor([-1.2] * 3)) and torch.allclose(m.xyz_max, torch.tensor([1.2] * 3))
    assert m.world_len == int(m.world_size[0]) and list(m.density.grid.shape) == [1, 1] + m.world_size.tolist()
    assert abs(float(m.act_shift) - np.log(1 / (1 - 1e-2) - 1)) < 1e-6
    keys = set(m.state_dict().keys())
    assert {'scene_center', 'scene_radius', 'xyz_min', 'xyz_max', 'act_shift', 'viewfreq', 'density.grid', 'k0.grid',
            'mask_cache.mask', 'rgbnet.0.weight', 'rgbnet.2.0.weight', 'rgbnet.3.bias'} <= keys
    assert m.rgbnet[0].in_features == 3 + 3 * 4 * 2 + 12
    kw = m.get_kwargs()
    assert kw['contracted_norm'] == 'inf' and kw['rgbnet_dim'] == 12 and kw['num_voxels'] == 40 ** 3
    t = m.sample_t(0.5, 'cpu')
    n_inner = int(2 / (2 + 2 * 0.2) * m.world_len / 0.5) + 1
    assert t.numel() == 2 * n_inner and bool((t[1:] > t[:-1]).all())
    assert abs(float(t[0]) - 1.0 / n_inner) < 1e-6 and float(t[-1]) > 100
    dvgo = k4nerf.DirectVoxGO([-1] * 3, [1] * 3, num_voxels=8 ** 3, num_voxels_base=8 ** 3, alpha_init=1e-2,
                              fast_color_thres=1e-4, rgbnet_dim=12)
    dmpigo = k4nerf.DirectMPIGO([-1] * 3, [1] * 3, num_voxels=8 ** 3, mpi_depth=8, fast_color_thres=1e-3, rgbnet_dim=9,
                                rgbnet_width=64, act_type='relu', mode_type='mlp')
    for km in (m, dvgo, dmpigo):                      # 'tc' / 'tcgen05' (K4_MLP_TCGEN05) alias the wgmma marcher 'ws'
        assert km.resolve_mlp_mode('tc') == km.resolve_mlp_mode('tcgen05') == 'ws' and km.resolve_mlp_mode('fp32') == 'fp32'
    with pytest.raises(RuntimeError):                 # 'auto' asks the library which kernels cover the DEVICE scene: no CPU path
        m.resolve_mlp_mode('auto')
    with pytest.raises(NotImplementedError):
        k4nerf.DirectContractedVoxGO(xyz_min=[-1] * 3, xyz_max=[1] * 3, num_voxels=8 ** 3, num_voxels_base=8 ** 3,
                                     alpha_init=1e-2, contracted_norm='l2')


def test_masked_adam_argument_validation_and_training_modules_import():
    """lib/masked_adam.py:19-30 argument checks; the drop-in module names of the reference's four CUDA
    extensions all exist with the reference's function names."""
    p = torch.nn.Parameter(torch.zeros(3))
    for bad in (dict(lr=-1.0), dict(eps=-1e-8), dict(betas=(1.0, 0.99)), dict(betas=(0.9, -0.1))):
        with pytest.raises(ValueError):
            k4nerf.MaskedAdam([p], **bad)
    opt = k4nerf.MaskedAdam([{'params': [p], 'skip_zero_grad': True}], lr=0.5)
    assert opt.per_lr is None and opt.param_groups[0]['lr'] == 0.5 and opt.param_groups[0]['betas'] == (0.9, 0.99)
    opt.step()                                                    # no grads: nothing to do, no GPU needed
    from k4nerf import render_utils_cuda, total_variation_cuda, adam_upd_cuda, ub360_utils_cuda, autograd_ops
    assert callable(total_variation_cuda.total_variation_add_grad) and callable(ub360_utils_cuda.cumdist_thres)
    assert {'adam_upd', 'masked_adam_upd', 'adam_upd_with_perlr'} <= set(dir(adam_upd_cuda))
    assert {'Raw2Alpha', 'Raw2Alpha_nonuni', 'Alphas2Weights'} <= set(dir(autograd_ops))
    assert issubclass(autograd_ops.Raw2Alpha, torch.autograd.Function)
    with pytest.raises(RuntimeError, match='CUDA'):
        adam_upd_cuda.adam_upd(torch.zeros(4), torch.zeros(4), torch.zeros(4), torch.zeros(4), 1, 0.9, 0.99, 0.1, 1e-8)
    assert len(render_utils_cuda.__doc__) > 0


def test_sftnet_save_network_round_trips_through_load_network(tmp_path):
    """lib/sr_esrnet.py:589-622 / :529-554: '<label>_<iter>.pth' with {'params': state_dict} on the CPU, -1 -> 'latest'."""
    torch.manual_seed(7)
    a = k4nerf.SFTNet(3, 4, 64, 1, 32, 1)
    path = a.save_network(str(tmp_path), 'net_sr', -1)
    assert path == os.path.join(str(tmp_path), 'net_sr_latest.pth') and os.path.exists(path)
    blob = torch.load(path, weights_only=False)
    assert list(blob) == ['params'] and all(not v.is_cuda for v in blob['params'].values())
    b = k4nerf.SFTNet(3, 4, 64, 1, 32, 1)
    b.load_network(path, 'cpu', strict=True, param_key='params')
    for (ka, va), (kb, vb) in zip(a.state_dict().items(), b.state_dict().items()):
        assert ka == kb and torch.equal(va, vb)
    assert a.save_network(str(tmp_path), 'net_sr', 1500).endswith('net_sr_1500.pth')


def test_render_viewpoints_dump_images_writes_the_reference_file_names(tmp_path):
    """run.py:161-165 / run_sr.py:171-175: e<global_step>_<index>.png of the 8-bit frames (after the video flip / rot90)."""
    import numpy as np
    from k4nerf import render
    rgbs = [np.random.RandomState(i).rand(6, 8, 3).astype(np.float32) * 1.2 - 0.1 for i in range(2)]
    render._dump(rgbs, str(tmp_path), True, 1500)
    assert sorted(os.listdir(tmp_path)) == ['e1500_000.png', 'e1500_001.png']
    from PIL import Image
    got = np.array(Image.open(os.path.join(tmp_path, 'e1500_001.png')))
    assert np.array_equal(got, render.to8b(rgbs[1]))
    render._dump(rgbs, None, True, 0)                  # no directory / not asked for: nothing happens
    render._dump(rgbs, str(tmp_path), False, 0)
    assert len(os.listdir(tmp_path)) == 2


def test_rgb_ssim_matches_the_windowed_definition():
    """utils.rgb_ssim (lib/utils.py:88-134) against a direct evaluation of the definition: 11x11 Gaussian window
    (sigma 1.5) at every 'valid' position, per channel."""
    import numpy as np
    from k4nerf.utils import rgb_ssim
    rs = np.random.RandomState(0)
    a = rs.rand(20, 23, 3)
    b = np.clip(a + 0.1 * rs.randn(20, 23, 3), 0, 1)
    assert abs(rgb_ssim(a, a, 1) - 1.0) < 1e-12
    t = np.arange(11) - 5
    g = np.exp(-0.5 * (t / 1.5) ** 2); g /= g.sum()
    w2 = np.outer(g, g)
    c1, c2 = 0.01 ** 2, 0.03 ** 2
    vals = []
    for y in range(20 - 10):
        for x in range(23 - 10):
            for c in range(3):
                p, q = a[y:y + 11, x:x + 11, c], b[y:y + 11, x:x + 11, c]
                m0, m1 = (w2 * p).sum(), (w2 * q).sum()
                v0 = max((w2 * p * p).sum() - m0 * m0, 0.0); v1 = max((w2 * q * q).sum() - m1 * m1, 0.0)
                cv = (w2 * p * q).sum() - m0 * m1
                cv = np.sign(cv) * min(np.sqrt(v0 * v1), abs(cv))
                vals.append((2 * m0 * m1 + c1) * (2 * cv + c2) / ((m0 * m0 + m1 * m1 + c1) * (v0 + v1 + c2)))
    got = rgb_ssim(a.astype(np.float32), b.astype(np.float32), max_val=1)
    assert abs(got - np.mean(vals)) < 1e-6 and 0 < got < 1
    assert rgb_ssim(a, b, 1, return_map=True).shape == (10, 13, 3)


@pytest.mark.parametrize('ndc', [False, True])
@pytest.mark.parametrize('mode', ['lefttop', 'center'])
def test_get_rays_of_a_view_torch_modes_match_the_oracle(ndc, mode):
    """lib/dvgo.py:516-582: the sub-pixel modes the device kernel does not generate run in plain torch; same values as
    the oracle's restatement (flips, inverse_y, NDC warp; view directions taken before the warp)."""
    from k4nerf import dvgo, coarse
    from oracle import pipeline as opipe, scenes
    H, W = 13, 17
    K, c2w = scenes.llff_camera(H, W, (0.05, -0.03, 0.0)) if ndc else scenes.blender_camera(H, W)
    for inv_y, fx, fy in ((False, False, False), (True, True, False), (False, False, True)):
        ref = opipe.get_rays_of_a_view(H, W, K, c2w, ndc, inv_y, fx, fy, mode=mode)
        got = coarse.get_rays_of_a_view_torch(H, W, K, c2w, ndc, inv_y, fx, fy, mode=mode)
        for a, b in zip(got, ref):
            assert a.shape == (H, W, 3) and torch.allclose(a, b, rtol=1e-6, atol=1e-6)
    if mode != 'center':        # the public entry point routes non-centre modes to the torch path (no GPU needed)
        got = dvgo.get_rays_of_a_view(H, W, K, c2w, ndc, False, False, False, mode=mode)
        ref = opipe.get_rays_of_a_view(H, W, K, c2w, ndc, False, False, False, mode=mode)
        assert all(torch.allclose(a, b, rtol=1e-6, atol=1e-6) for a, b in zip(got, ref))
    r = dvgo.get_rays_of_a_view(H, W, K, c2w, ndc, False, False, False, mode='random')
    lo = opipe.get_rays_of_a_view(H, W, K, c2w, False, False, False, False, mode='lefttop')
    assert r[0].shape == (H, W, 3) and torch.isfinite(r[1]).all() and lo[0].shape == (H, W, 3)
