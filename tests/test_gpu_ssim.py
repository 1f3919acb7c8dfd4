"""GPU: utils.rgb_ssim of CUDA tensors (k4_op_rgb_ssim, csrc/k4_metrics.cu) against the numpy path, at small, LR-frame
and 4K sizes and on the reference's golden cases; strided views read in place; bitwise determinism; the eval_ssim
option of render_viewpoints / render_viewpoints_sr; and the errors of both layers."""
import ctypes as C
import os

import numpy as np
import pytest
import torch

from k4nerf import render
from k4nerf.utils import rgb_ssim
from helpers import make_state, model_from_state
from oracle import scenes

pytestmark = pytest.mark.gpu

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden', 'ssim_ref.pt')


def _pair(H, W, seed, dtype=torch.float32):
    """A smooth image and a noisy copy in [0, 1] (so that the map spans a range of values), on the CPU."""
    g = torch.Generator().manual_seed(seed)
    a = torch.rand(1, 3, H, W, generator=g, dtype=torch.float64)
    a = torch.nn.functional.avg_pool2d(a, 3, stride=1, padding=1, count_include_pad=False)[0].permute(1, 2, 0)
    b = (a + 0.1 * torch.randn(H, W, 3, generator=g, dtype=torch.float64)).clamp(0, 1)
    return a.to(dtype).contiguous(), b.to(dtype).contiguous()


def _check_against_numpy(a, b, dev, mean_tol=1e-12, map_tol=1e-11, **kw):
    ref_map = rgb_ssim(a.numpy(), b.numpy(), return_map=True, **kw)
    ref_mean = rgb_ssim(a.numpy(), b.numpy(), **kw)
    got_map = rgb_ssim(a.to(dev), b.to(dev), return_map=True, **kw)
    got_mean = rgb_ssim(a.to(dev), b.to(dev), **kw)
    assert isinstance(got_mean, float)
    assert got_map.is_cuda and got_map.dtype == torch.float64 and tuple(got_map.shape) == ref_map.shape
    assert got_map.is_contiguous()
    assert np.abs(got_map.cpu().numpy() - ref_map).max() <= map_tol
    assert abs(got_mean - ref_mean) <= mean_tol, (got_mean, ref_mean)
    return got_mean


@pytest.mark.parametrize('dtype', [torch.float32, torch.float64])
@pytest.mark.parametrize('H,W', [(11, 11), (12, 37), (757, 1009)])
def test_matches_the_numpy_path(cuda_device, H, W, dtype):
    a, b = _pair(H, W, seed=H * 1000 + W, dtype=dtype)
    _check_against_numpy(a, b, cuda_device, max_val=1)


def test_matches_the_numpy_path_on_a_4k_frame(cuda_device):
    """One 4032 x 3024 fp32 pair: 11970 tiles, the mean summed over all of them."""
    a, b = _pair(3024, 4032, seed=4, dtype=torch.float32)
    ref_map = rgb_ssim(a.numpy(), b.numpy(), return_map=True, max_val=1)
    got_map = rgb_ssim(a.to(cuda_device), b.to(cuda_device), 1, return_map=True)
    assert np.abs(got_map.cpu().numpy() - ref_map).max() <= 1e-11
    assert abs(rgb_ssim(a.to(cuda_device), b.to(cuda_device), 1) - float(ref_map.mean())) <= 1e-12


@pytest.mark.parametrize('name', sorted(torch.load(GOLD, map_location='cpu', weights_only=False)['cases']))
def test_matches_the_reference_golden(cuda_device, name):
    """The reference's own rgb_ssim (fp64 pairs): every map element within 1e-11, the mean within 1e-12 of the numpy
    path's."""
    c = torch.load(GOLD, map_location='cpu', weights_only=False)['cases'][name]
    kw = c['kwargs']
    got = rgb_ssim(c['img0'].to(cuda_device), c['img1'].to(cuda_device), return_map=True, **kw)
    assert np.abs(got.cpu().numpy() - c['map'].numpy()).max() <= 1e-11
    _check_against_numpy(c['img0'], c['img1'], cuda_device, **kw)


def test_promotes_other_dtypes_to_fp64(cuda_device):
    """u8 and fp16 images and a mixed fp32 / fp64 pair are widened to fp64 (exactly, as numpy's asarray)."""
    a, b = _pair(40, 52, seed=8, dtype=torch.float64)
    a8, b8 = (a * 255).round().to(torch.uint8), (b * 255).round().to(torch.uint8)
    _check_against_numpy(a8, b8, cuda_device, max_val=255)
    _check_against_numpy(a.half(), b.half(), cuda_device, max_val=1)
    _check_against_numpy(a.float(), b, cuda_device, max_val=1)
    _check_against_numpy(a.half(), b.float(), cuda_device, max_val=1)


@pytest.mark.parametrize('dtype', [torch.float32, torch.float64])
def test_strided_views_are_read_in_place(cuda_device, dtype):
    """A CHW frame through permute(1, 2, 0), a crop and an expanded constant image: bit-identical to their
    contiguous copies."""
    dev = cuda_device
    a, b = _pair(90, 70, seed=9, dtype=dtype)
    chw = b.permute(2, 0, 1).contiguous().to(dev)             # [3, H, W], as render_frame_4k's sr
    view = chw.permute(1, 2, 0)
    assert not view.is_contiguous()
    big = torch.rand(120, 110, 3, dtype=dtype, generator=torch.Generator().manual_seed(1)).to(dev)
    crop = big[13:103, 21:91]
    const = torch.tensor([0.25, 0.5, 0.75], dtype=dtype, device=dev).expand(90, 70, 3)
    assert const.stride() == (0, 0, 1)
    a = a.to(dev)
    for v in (view, crop, const):
        cpy = v.contiguous()
        for x0, x1, y0, y1 in ((a, v, a, cpy), (v, a, cpy, a)):
            assert torch.equal(rgb_ssim(x0, x1, 1, return_map=True), rgb_ssim(y0, y1, 1, return_map=True))
            assert rgb_ssim(x0, x1, 1) == rgb_ssim(y0, y1, 1)


def test_deterministic_and_one_on_identical_images(cuda_device):
    a, b = _pair(300, 410, seed=10)
    a, b = a.to(cuda_device), b.to(cuda_device)
    assert torch.equal(rgb_ssim(a, b, 1, return_map=True), rgb_ssim(a, b, 1, return_map=True))
    assert rgb_ssim(a, b, 1) == rgb_ssim(a, b, 1)
    assert abs(rgb_ssim(a, a, 1) - 1.0) <= 1e-12
    assert abs(rgb_ssim(b, b.clone(), 1) - 1.0) <= 1e-12


def _scene(dev):
    m = model_from_state(make_state('cfgA', res=32, regime='fog'), dev)
    m.mlp_mode = 'fp32'                                # sequential per-ray accumulation: frames reproduce bit for bit
    H, W = 30, 44
    poses, Ks = [], []
    for th in (30.0, 120.0):
        K, c2w = scenes.blender_camera(H, W, theta=th)
        poses.append(c2w.numpy()); Ks.append(K)
    rng = np.random.default_rng(5)
    gt = [np.clip(0.5 + 0.3 * rng.standard_normal((H, W, 3)), 0, 1).astype(np.float32) for _ in range(2)]
    return m, np.array(poses), np.array([[H, W]] * 2), np.array(Ks), gt


def test_render_viewpoints_scores_on_the_device(cuda_device, monkeypatch):
    """eval_ssim scores the clamped frame on the device; the SSIM values are the numpy path's on the returned frames
    within 1e-12, and PSNR and the arrays are those of a run without it."""
    m, poses, HW, Ks, gt = _scene(cuda_device)
    kw = dict(scenes.RENDER_KW_DVGO)
    seen = []
    real = render.rgb_ssim

    def spy(img0, img1, max_val, **k):
        seen.append((img0.device, img1.device))
        return real(img0, img1, max_val, **k)
    monkeypatch.setattr(render, 'rgb_ssim', spy)
    on = render.render_viewpoints(m, poses, HW, Ks, False, kw, gt_imgs=gt, eval_ssim=True)
    off = render.render_viewpoints(m, poses, HW, Ks, False, kw, gt_imgs=gt, eval_ssim=False)
    assert seen == [(cuda_device, cuda_device)] * 2
    for x, y in zip(on[:3], off[:3]):
        assert np.array_equal(x, y)
    assert on[3] == off[3] and len(on[3]) == 2 and off[4] == []
    for i in range(2):
        assert isinstance(on[4][i], float)
        assert abs(on[4][i] - rgb_ssim(on[0][i], gt[i], max_val=1)) <= 1e-12


def test_render_viewpoints_sr_scores_on_the_device(cuda_device, capsys):
    """run_sr.py's variant prints the mean SSIM (it does not return it): the numpy path's value within 1e-12."""
    m, poses, HW, Ks, gt = _scene(cuda_device)
    kw = dict(scenes.RENDER_KW_DVGO)
    capsys.readouterr()
    on = render.render_viewpoints_sr(m, poses, HW, Ks, False, kw, gt_imgs=gt, eval_ssim=True)
    lines = capsys.readouterr().out.splitlines()
    off = render.render_viewpoints_sr(m, poses, HW, Ks, False, kw, gt_imgs=gt, eval_ssim=False)
    printed = [float(l.split()[2]) for l in lines if l.startswith('Testing ssim')]
    assert len(printed) == 1
    want = np.mean([rgb_ssim(on[0][i], gt[i], max_val=1) for i in range(2)])
    assert abs(printed[0] - want) <= 1e-12
    for i in (0, 1, 2, 5):
        assert np.array_equal(on[i], off[i])
    assert on[3] == off[3]


def test_errors(cuda_device):
    dev = cuda_device
    a, b = _pair(20, 24, seed=12)
    with pytest.raises(AssertionError):
        rgb_ssim(a.to(dev), b[:, :-1].to(dev), 1)
    with pytest.raises(AssertionError):
        rgb_ssim(a[..., :2].to(dev), b[..., :2].to(dev), 1)
    with pytest.raises(AssertionError):
        rgb_ssim(a[0].to(dev), b[0].to(dev), 1)
    with pytest.raises(ValueError):
        rgb_ssim(a[:10].to(dev), b[:10].to(dev), 1)                 # 10 rows < the 11-tap window
    with pytest.raises(ValueError):
        rgb_ssim(a.to(dev), b.to(dev), 1, filter_size=32)
    with pytest.raises(RuntimeError):
        rgb_ssim(a.to(dev), b, 1)
    with pytest.raises(RuntimeError):
        rgb_ssim(a.numpy(), b.to(dev), 1)
    # CPU tensors still take the numpy path
    assert rgb_ssim(a, b, 1) == rgb_ssim(a.numpy(), b.numpy(), 1)
    assert isinstance(rgb_ssim(a, b, 1, return_map=True), np.ndarray)


def test_short_workspace_is_reported(cuda_device):
    """The C ABI with real device buffers: one byte short of the workspace size is K4_ERR_WORKSPACE, nothing runs."""
    from k4nerf import _lib
    dev = cuda_device
    a, b = (t.to(dev) for t in _pair(64, 64, seed=13))
    need = _lib.lib.k4_op_rgb_ssim_workspace_bytes(64, 64, 11)
    ws = torch.zeros(need, dtype=torch.uint8, device=dev)
    mean = torch.full((), -7.0, dtype=torch.float64, device=dev)
    st = (C.c_int64 * 3)(*a.stride())
    win = (C.c_double * 11)(*([1.0 / 11] * 11))

    def call(nbytes):
        return _lib.lib.k4_op_rgb_ssim(C.c_void_p(a.data_ptr()), C.c_void_p(b.data_ptr()), 0, 64, 64, st, st, win, 11, 1e-4,
                                       9e-4, None, C.c_void_p(mean.data_ptr()), C.c_void_p(ws.data_ptr()), nbytes,
                                       C.c_void_p(torch.cuda.current_stream(dev).cuda_stream))
    assert call(need - 1) == -4
    torch.cuda.synchronize()
    assert mean.item() == -7.0
    assert call(need) == 0
    torch.cuda.synchronize()
    assert -1 <= mean.item() <= 1
