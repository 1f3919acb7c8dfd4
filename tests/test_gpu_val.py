"""GPU: the joint stage's validation on the device (csrc/k4_val.cu; utils.resize_quarter / rgb_mse,
render.render_val_4k) -- the resize bit for bit against the cv2 golden and the numpy restatement, in place on strided,
permuted and cropped views; the MSE and PSNR bit for bit against numpy on both layouts from 1x1 to 4K, identical
frames, NaN and inf, repeated calls; and render_val_4k against a literal transcription of run_sr.py:1088-1146."""
import io
import os

import numpy as np
import pytest
import torch

import k4nerf
from k4nerf import render, utils
from k4nerf.utils import resize_quarter, rgb_lpips, rgb_mse, to8b
from helpers import make_state, model_from_state
from oracle import lpips as lpips_ref, scenes, sftnet
from val_ref import mse_np

pytestmark = pytest.mark.gpu
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden', 'resize_quarter_ref.pt')


def test_resize_matches_the_cv2_golden(cuda_device):
    for c in torch.load(GOLDEN, weights_only=False)['cases']:
        got = resize_quarter(c['x'].to(cuda_device))
        assert got.is_contiguous() and torch.equal(got.cpu(), c['out']), (c['H'], c['W'])


@pytest.mark.parametrize('H,W', [(3, 3), (3, 10), (10, 3), (5, 6), (758, 1010), (757, 1011), (3024, 4032)])
def test_resize_views_match_the_restatement(cuda_device, H, W):
    g = torch.Generator().manual_seed(H + W)
    planes = torch.rand(3, H, W, generator=g)
    views = {'planar': planes.movedim(0, -1), 'contiguous': planes.movedim(0, -1).contiguous(),
             'transposed': torch.rand(W, H, 3, generator=g).transpose(0, 1),
             'cropped': torch.rand(H + 3, W + 2, 5, generator=g)[2:-1, 1:-1, 1:4]}
    for name, v in views.items():
        want = utils._resize_quarter_np(v.numpy())
        got = resize_quarter(v.to(cuda_device))
        assert np.array_equal(got.cpu().numpy(), want), name


def _pair(H, W, layout, seed):
    g = torch.Generator().manual_seed(seed)
    if layout == 'planar':                                   # run_sr.py:768 / 1131: movedim views of [3, H, W] planes
        return [torch.rand(1, 3, H, W, generator=g).squeeze(0).movedim(0, -1) for _ in range(2)]
    return [torch.rand(H, W, 3, generator=g) for _ in range(2)]


@pytest.mark.parametrize('layout', ['planar', 'contiguous'])
@pytest.mark.parametrize('H,W', [(1, 1), (1, 5), (3, 2), (7, 9), (43, 16), (189, 252), (756, 1008), (2897, 2001),
                                 (3024, 4032)])
def test_mse_and_psnr_are_numpys(cuda_device, layout, H, W):
    a, b = _pair(H, W, layout, H * 7 + W)
    want = np.mean(np.square(a.numpy() - b.numpy()))
    got = rgb_mse(a.to(cuda_device), b.to(cuda_device))
    assert type(got) is np.float32 and got == want and mse_np(a.numpy(), b.numpy()) == want
    assert -10. * np.log10(got) == -10. * np.log10(want)
    assert rgb_mse(a.to(cuda_device), b.to(cuda_device)) == got                  # repeated calls: the same bits


def test_mse_mixed_layouts_and_special_values(cuda_device):
    a, b = _pair(64, 80, 'planar', 1)
    c = b.contiguous()
    for x, y in ((a, c), (c, a), (a, a)):
        assert rgb_mse(x.to(cuda_device), y.to(cuda_device)) == np.mean(np.square(x.numpy() - y.numpy()))
    with np.errstate(divide='ignore'):
        assert np.isinf(-10. * np.log10(rgb_mse(a.to(cuda_device), a.to(cuda_device))))
    x = a.clone()
    x[3, 4, 1] = float('inf')
    assert rgb_mse(x.to(cuda_device), b.to(cuda_device)) == np.inf
    x[5, 6, 2] = float('nan')
    assert np.isnan(rgb_mse(x.to(cuda_device), b.to(cuda_device)))
    y = b.clone()
    y[3, 4, 1] = float('inf')
    assert np.isnan(rgb_mse(x.to(cuda_device), y.to(cuda_device)))                # inf - inf
    with pytest.raises(TypeError):
        rgb_mse(a.double().to(cuda_device), b.double().to(cuda_device))
    with pytest.raises(RuntimeError):
        rgb_mse(a.to(cuda_device), b.numpy())


# ---- render_val_4k ----------------------------------------------------------------------------------------------
H, W, N = 24, 32, 2


def _decode(path):
    from PIL import Image
    return np.asarray(Image.open(io.BytesIO(path.read_bytes())).convert('RGB'))


def _host_resize(x):
    try:
        import cv2
    except ImportError:
        return utils._resize_quarter_np(x)
    return cv2.resize(x, dsize=None, fx=1 / 4, fy=1 / 4)


def _reference_block(m, net, poses, HW, Ks, kw, gt, srgt, load_sr, savedir, weights, dev, test_tile, sel_b=0, step=5):
    """run_sr.py:1088-1146, line for line, with render_viewpoints_sr, tile_process to the CPU and numpy / cv2 scores."""
    from k4nerf.sr_esrnet import sft_condition
    rgbs, depths, bgmaps, psnrs_test, viewdirs, rgb_features = render.render_viewpoints_sr(
        m, poses, HW, Ks, False, kw, gt_imgs=gt, savedir=savedir, global_step=step)
    out = []
    for idx, rgbsave in enumerate(rgb_features):
        rgbtest = torch.from_numpy(rgbsave).movedim(-1, 0).unsqueeze(0).to(dev)
        input_cond = sft_condition(net.num_cond, torch.from_numpy(depths[idx]).to(dev), viewdirs[idx], H, W)
        rgb_srtest = net.tile_process(rgbtest, input_cond, tile_size=test_tile)
        render._write_png(os.path.join(savedir, f'test_{step}.png'), to8b(rgbs[idx]))
        rgb_srsave = rgb_srtest.squeeze().movedim(0, -1).detach().clamp(0, 1).cpu().numpy()
        sr_mse = np.mean(np.square(rgb_srsave - srgt[idx]))
        sr_psnr = -10. * np.log10(sr_mse)
        sr_ssim = utils.rgb_ssim(rgb_srsave, srgt[idx], max_val=1)
        if load_sr == 1:
            sr_lpips = rgb_lpips(_host_resize(rgb_srsave), _host_resize(srgt[idx]), 'vgg', device=dev, weights=weights)
        else:
            sr_lpips = rgb_lpips(rgb_srsave, srgt[idx], 'vgg', device=dev, weights=weights)
        render._write_png(os.path.join(savedir, f'testsr_{step}_{sel_b}.png'), to8b(rgb_srsave))
        out.append((sr_psnr, sr_ssim, sr_lpips, to8b(rgbs[idx]), to8b(rgb_srsave)))
    return (rgbs, depths, bgmaps, psnrs_test, viewdirs, rgb_features), out


@pytest.fixture(scope='module')
def scene(cuda_device):
    m = model_from_state(make_state('cfgA', res=32, regime='shell'), cuda_device)
    m.mlp_mode = 'fp32'
    poses, Ks = [], []
    for th in (30.0, 100.0):
        K, c2w = scenes.blender_camera(H, W, theta=th)
        poses.append(c2w.numpy()); Ks.append(K)
    return m, np.array(poses), np.array([[H, W]] * N), np.array(Ks), dict(scenes.RENDER_KW_DVGO)


@pytest.mark.parametrize('scale,nc,load_sr', [(4, 1, 1), (4, 63, 1), (4, 64, 1), (1, 1, 4)])
def test_render_val_4k_is_the_host_block(scene, cuda_device, tmp_path, capsys, scale, nc, load_sr):
    m, poses, HW, Ks, kw = scene
    net = k4nerf.SFTNet(3, scale, 64, 5, 32, nc)
    sd = sftnet.random_state_dict(seed=3, num_cond=nc)
    if scale == 1:
        sd = {k: v for k, v in sd.items() if not k.startswith(('conv_up1.', 'conv_up2.'))}
    net.load_state_dict(sd)
    net = net.to(cuda_device)
    weights = lpips_ref.random_state_dict('vgg', seed=1)
    g = torch.Generator().manual_seed(11)
    gt = [torch.rand(H, W, 3, generator=g).numpy() for _ in range(N)]
    # rgb_srgt_val as run_sr.py:765-769 builds it: [N, 3, sH, sW] planes viewed as [N, sH, sW, 3]
    srgt = torch.rand(N, 3, scale * H, scale * W, generator=g).movedim(1, -1).numpy()
    want_dir, got_dir = tmp_path / 'want', tmp_path / 'got'
    want_dir.mkdir(); got_dir.mkdir()
    want_lr, want = _reference_block(m, net, poses, HW, Ks, kw, gt, srgt, load_sr, str(want_dir), weights, cuda_device, 16)
    capsys.readouterr()
    got = render.render_val_4k(m, net, poses, HW, Ks, False, kw, gt, srgt, load_sr, savedir=str(got_dir), global_step=5,
                               test_tile=16, lpips_weights=weights)
    printed = capsys.readouterr().out
    for i in (0, 1, 2, 5):
        assert got[i].dtype == want_lr[i].dtype and np.array_equal(got[i], want_lr[i]), i
    assert got[3] == want_lr[3]
    assert all(torch.equal(a, b) for a, b in zip(got[4], want_lr[4]))
    sr_psnrs, sr_ssims, sr_lpips = got[6:]
    for i, (p, s, l, _, _) in enumerate(want):
        assert type(sr_psnrs[i]) is type(p) is np.float32 and sr_psnrs[i] == p, i
        assert abs(sr_ssims[i] - s) <= 1e-12, (sr_ssims[i], s)
        assert sr_lpips[i] == l, (sr_lpips[i], l)
        assert f'Testing psnr {p!s} (sr)' in printed and f'Testing lpips {l!s} (sr)' in printed
    # the files hold the last view, as the reference's overwritten ones
    assert sorted(os.listdir(got_dir)) == ['test_5.png', 'testsr_5_0.png']
    for name, k in (('test_5.png', 3), ('testsr_5_0.png', 4)):
        assert np.array_equal(_decode(got_dir / name), want[-1][k])
        assert np.array_equal(_decode(got_dir / name), _decode(want_dir / name))


def test_render_val_4k_takes_cuda_ground_truth(scene, cuda_device):
    m, poses, HW, Ks, kw = scene
    net = k4nerf.SFTNet(3, 4, 64, 5, 32, 1)
    net.load_state_dict(sftnet.random_state_dict(seed=3))
    net = net.to(cuda_device)
    weights = lpips_ref.random_state_dict('vgg', seed=1)
    srgt = torch.rand(N, 3, 4 * H, 4 * W, generator=torch.Generator().manual_seed(2)).movedim(1, -1)
    a = render.render_val_4k(m, net, poses, HW, Ks, False, kw, None, srgt.numpy(), 1, test_tile=16, lpips_weights=weights)
    b = render.render_val_4k(m, net, poses, HW, Ks, False, kw, None, srgt.to(cuda_device), 1, test_tile=16,
                             lpips_weights=weights)
    assert a[6:] == b[6:] and a[3] == b[3] == []
